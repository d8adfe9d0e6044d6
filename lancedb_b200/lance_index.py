"""Reading an on-disk Lance IVF_PQ index (``<table>.lance/_indices/<uuid>/{index.idx,auxiliary.idx}``) into the
plain arrays of ``lgpu_index_desc`` (SURVEY.md 8f-3).

STATUS: **[lance, recalled] -- UNVERIFIED against a real file.**  The reference tree holds no Lance index file and no
Lance writer (the file format lives in the un-vendored lance crates, v11.0.0-beta.19; the only thing
the reference pins is that the directory ``_indices/<uuid>/`` exists: nodejs/__test__/table.test.ts:907, 1318).
The layout below is the Lance v2 file container + the v3 vector-index layout as published in lance's
``protos/file2.proto``, ``protos/encodings.proto`` and ``protos/index.proto``, restated from memory:

  file      := data pages | column metadata blobs | column-metadata offset table | global-buffer offset table | footer
  footer    := u64 col_meta_start, u64 cmo_table_off, u64 gbo_table_off, u32 n_global_buffers, u32 n_columns,
               u16 major, u16 minor, "LANC"                                                  (40 bytes, little endian)
  CMO / GBO := n x (u64 position, u64 size)
  global buffer 0 := FileDescriptor { schema = 1 { fields = 1 [Field], metadata = 5 map<string,bytes> }, length = 2 }
  column metadata := ColumnMetadata { encoding = 1, pages = 2 [Page{buffer_offsets = 1, buffer_sizes = 2, length = 3,
                     encoding = 4}], buffer_offsets = 3, buffer_sizes = 4 };  Page.encoding = Encoding{direct = 2
                     {encoding = 1: bytes of google.protobuf.Any{type_url = 1, value = 2: ArrayEncoding}}}
  ArrayEncoding   := flat = 1 {bits_per_value = 1, buffer = 2 {buffer_index = 1, buffer_type = 2}} |
                     nullable = 2 {no_nulls = 1 {values = 1}} | fixed_size_list = 3 {dimension = 1, items = 2}
  index.idx       schema metadata: "lance:index" = {"type": "IVF_PQ", "distance_type": "l2"},
                  "lance:ivf" = index of the global buffer holding pb IVF {offsets = 2, lengths = 3,
                  centroids_tensor = 4 {data_type = 1 (FLOAT32 = 2), shape = 2, data = 3}}
  auxiliary.idx   columns ``_rowid`` u64 and ``__pq_code`` fixed_size_list<u8>[m]; schema metadata "lance:ivf" as above
                  (the partition offsets / lengths of THIS file's rows), "storage_metadata" = JSON list with one JSON
                  string {"codebook_position": g, "nbits": 8, "num_sub_vectors": m, "dimension": d,
                  "transposed": bool}; global buffer g = pb Tensor of the codebook, f32 [256, d] laid out
                  codebook[c][i * dsub + t]; transposed = the codes of a partition are stored column-major
                  ([m][n_p], SURVEY.md 8a row a6).

Only the subset above is handled (flat, non-null, uncompressed pages -- what an index file needs); anything else
raises ``LanceFormatError`` naming the unsupported piece, so a real file that deviates from the recollection fails
loudly instead of loading garbage.  ``write_ivf_pq_index`` emits the same layout: it exists for the round-trip tests
and as an executable statement of the recollection, not as a Lance writer.

Host side only, no GPU work: the arrays feed ``IvfPqIndexData`` -> ``lgpu_index_open`` exactly like the in-memory
build (lancedb_b200/index.py); the kernels never see the file format.
"""
from __future__ import annotations

import json
import os
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

MAGIC = b"LANC"
FOOTER_LEN = 40
ANY_ARRAY_ENCODING = "/lance.encodings.ArrayEncoding"
TENSOR_F32 = 2          # pb Tensor.DataType: BFLOAT16 = 0, FLOAT16 = 1, FLOAT32 = 2, FLOAT64 = 3


class LanceFormatError(ValueError):
    pass


# ------------------------------------------------------------------------------------------ protobuf wire format
def _varint(buf: bytes, pos: int) -> Tuple[int, int]:
    out = shift = 0
    while True:
        if pos >= len(buf):
            raise LanceFormatError("truncated varint")
        b = buf[pos]
        pos += 1
        out |= (b & 0x7F) << shift
        if not b & 0x80:
            return out, pos
        shift += 7
        if shift > 63:
            raise LanceFormatError("varint longer than 64 bits")


def pb_fields(buf: bytes) -> Dict[int, list]:
    """Decode one message into {field number: [raw values]}: ints for varint / fixed, bytes for length-delimited."""
    out: Dict[int, list] = {}
    pos = 0
    while pos < len(buf):
        key, pos = _varint(buf, pos)
        fno, wt = key >> 3, key & 7
        if wt == 0:
            v, pos = _varint(buf, pos)
        elif wt == 1:
            v = struct.unpack_from("<Q", buf, pos)[0]
            pos += 8
        elif wt == 2:
            n, pos = _varint(buf, pos)
            if pos + n > len(buf):
                raise LanceFormatError("truncated length-delimited field")
            v = bytes(buf[pos:pos + n])
            pos += n
        elif wt == 5:
            v = struct.unpack_from("<I", buf, pos)[0]
            pos += 4
        else:
            raise LanceFormatError(f"unsupported protobuf wire type {wt}")
        out.setdefault(fno, []).append(v)
    return out


def pb_repeated_ints(values: list) -> List[int]:
    """A repeated scalar field: packed (one bytes blob of varints) or unpacked (one entry per element)."""
    out: List[int] = []
    for v in values:
        if isinstance(v, (bytes, bytearray)):
            pos = 0
            while pos < len(v):
                x, pos = _varint(v, pos)
                out.append(x)
        else:
            out.append(int(v))
    return out


def _enc_varint(x: int) -> bytes:
    out = bytearray()
    while True:
        b = x & 0x7F
        x >>= 7
        if x:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def pb_int(fno: int, x: int) -> bytes:
    return _enc_varint(fno << 3) + _enc_varint(int(x))


def pb_bytes(fno: int, b: bytes) -> bytes:
    return _enc_varint((fno << 3) | 2) + _enc_varint(len(b)) + bytes(b)


def pb_packed(fno: int, xs) -> bytes:
    return pb_bytes(fno, b"".join(_enc_varint(int(x)) for x in xs))


# ------------------------------------------------------------------------------------------ the v2 file container
class LanceFile:
    """Footer, global buffers, schema metadata and flat column pages of one Lance v2 file."""

    def __init__(self, path: str):
        self.path = path
        with open(path, "rb") as f:
            self.data = f.read()
        d = self.data
        if len(d) < FOOTER_LEN or d[-4:] != MAGIC:
            raise LanceFormatError(f"{path}: not a Lance v2 file (no LANC magic)")
        (self.col_meta_start, cmo_off, gbo_off, n_gb, n_col, self.major, self.minor) = struct.unpack_from(
            "<QQQIIHH", d, len(d) - FOOTER_LEN)
        if self.major != 2 and (self.major, self.minor) != (0, 3):     # 2.x; "0.3" was the first v2 marker
            raise LanceFormatError(f"{path}: file format version {self.major}.{self.minor} is not v2")
        if self.major == 2 and self.minor >= 1:
            raise LanceFormatError(f"{path}: format 2.{self.minor} page layouts (mini-block / full-zip) are not handled")
        end = len(d) - FOOTER_LEN
        if not (cmo_off <= gbo_off <= end and cmo_off + 16 * n_col <= end and gbo_off + 16 * n_gb <= end):
            raise LanceFormatError(f"{path}: offset tables out of range")
        self.columns = [struct.unpack_from("<QQ", d, cmo_off + 16 * i) for i in range(n_col)]
        self.global_buffers = [struct.unpack_from("<QQ", d, gbo_off + 16 * i) for i in range(n_gb)]
        for pos, size in self.columns + self.global_buffers:
            if pos + size > end:
                raise LanceFormatError(f"{path}: a buffer runs past the footer")
        if n_gb < 1:
            raise LanceFormatError(f"{path}: no schema buffer")
        fd = pb_fields(self.global_buffer(0))
        schema = pb_fields(fd.get(1, [b""])[0])
        self.num_rows = int(fd.get(2, [0])[0])
        self.field_names: List[str] = []
        for fb in schema.get(1, []):
            fld = pb_fields(fb)
            # Field { type = 1, name = 2, id = 3, parent_id = 4, logical_type = 5, ... }: only top-level fields own a column
            if int(fld.get(4, [0xFFFFFFFFFFFFFFFF])[0]) in (0xFFFFFFFFFFFFFFFF, 0xFFFFFFFF) or 4 not in fld:
                self.field_names.append(fld.get(2, [b""])[0].decode())
        self.metadata: Dict[str, bytes] = {}
        for ent in schema.get(5, []):
            kv = pb_fields(ent)
            self.metadata[kv.get(1, [b""])[0].decode()] = kv.get(2, [b""])[0]

    def global_buffer(self, i: int) -> bytes:
        if not 0 <= i < len(self.global_buffers):
            raise LanceFormatError(f"{self.path}: global buffer {i} does not exist")
        pos, size = self.global_buffers[i]
        return self.data[pos:pos + size]

    def meta_json(self, key: str):
        if key not in self.metadata:
            raise LanceFormatError(f"{self.path}: schema metadata '{key}' is missing")
        return json.loads(self.metadata[key].decode())

    # ---- columns
    @staticmethod
    def _array_encoding(page_encoding: bytes) -> Dict[int, list]:
        enc = pb_fields(page_encoding)
        if 2 not in enc:
            raise LanceFormatError("page encoding is not stored inline (deferred encodings are not handled)")
        any_msg = pb_fields(pb_fields(enc[2][0]).get(1, [b""])[0])
        url = any_msg.get(1, [b""])[0].decode()
        if not url.endswith(ANY_ARRAY_ENCODING):
            raise LanceFormatError(f"page encoding '{url}' is not an ArrayEncoding (format 2.1 layouts are not handled)")
        return pb_fields(any_msg.get(2, [b""])[0])

    @classmethod
    def _flat_leaf(cls, arr: Dict[int, list]) -> Tuple[int, int, int]:
        """Walk nullable(no_nulls) / fixed_size_list down to the flat leaf: (bits per value, items per row, buffer)."""
        per_row = 1
        while True:
            if 1 in arr:                                   # flat
                flat = pb_fields(arr[1][0])
                if 3 in flat and pb_fields(flat[3][0]).get(1, [b""])[0] not in (b"", b"none"):
                    raise LanceFormatError("compressed flat pages are not handled")
                buf = pb_fields(flat.get(2, [b""])[0])
                if int(buf.get(2, [0])[0]) != 0:
                    raise LanceFormatError("only page-level buffers are handled")
                return int(flat.get(1, [0])[0]), per_row, int(buf.get(1, [0])[0])
            if 2 in arr:                                   # nullable
                nn = pb_fields(arr[2][0])
                if 1 not in nn:
                    raise LanceFormatError("pages with nulls are not handled (index columns are non-null)")
                arr = pb_fields(pb_fields(nn[1][0]).get(1, [b""])[0])
            elif 3 in arr:                                 # fixed_size_list
                fsl = pb_fields(arr[3][0])
                per_row *= int(fsl.get(1, [0])[0])
                arr = pb_fields(fsl.get(2, [b""])[0])
            else:
                raise LanceFormatError(f"array encoding with fields {sorted(arr)} is not handled")

    def read_flat_column(self, name: str, dtype, per_row: int = 1) -> np.ndarray:
        """All pages of a fixed-width column as one array of shape [rows] or [rows, per_row]."""
        if name not in self.field_names:
            raise LanceFormatError(f"{self.path}: no column '{name}' (have {self.field_names})")
        pos, size = self.columns[self.field_names.index(name)]
        cm = pb_fields(self.data[pos:pos + size])
        dtype = np.dtype(dtype)
        parts = []
        for pb in cm.get(2, []):
            page = pb_fields(pb)
            offs, sizes = pb_repeated_ints(page.get(1, [])), pb_repeated_ints(page.get(2, []))
            nrows = int(page.get(3, [0])[0])
            bits, items, bufi = self._flat_leaf(self._array_encoding(page.get(4, [b""])[0]))
            if bits != dtype.itemsize * 8 or items != per_row:
                raise LanceFormatError(f"{self.path}: column '{name}' is {items} x {bits}-bit per row, expected "
                                       f"{per_row} x {dtype.itemsize * 8}")
            if bufi >= len(offs):
                raise LanceFormatError(f"{self.path}: page buffer {bufi} missing")
            need = nrows * per_row * dtype.itemsize
            if sizes[bufi] < need or offs[bufi] + need > len(self.data):
                raise LanceFormatError(f"{self.path}: page of column '{name}' is shorter than its row count")
            parts.append(np.frombuffer(self.data, dtype, nrows * per_row, offs[bufi]))
        out = np.concatenate(parts) if parts else np.zeros(0, dtype)
        if out.shape[0] != self.num_rows * per_row:
            raise LanceFormatError(f"{self.path}: column '{name}' holds {out.shape[0] // per_row} rows, file says {self.num_rows}")
        return out.reshape(-1, per_row) if per_row > 1 else out


def _tensor_f32(buf: bytes, what: str) -> np.ndarray:
    t = pb_fields(buf)
    if int(t.get(1, [0])[0]) != TENSOR_F32:
        raise LanceFormatError(f"{what}: tensor data type {t.get(1, [0])[0]} (only FLOAT32 is handled)")
    shape = pb_repeated_ints(t.get(2, []))
    data = t.get(3, [b""])[0]
    n = int(np.prod(shape)) if shape else 0
    if len(data) != 4 * n:
        raise LanceFormatError(f"{what}: tensor of shape {shape} with {len(data)} data bytes")
    return np.frombuffer(data, np.float32).reshape(shape).copy()


def _ivf_model(f: LanceFile) -> Tuple[Optional[np.ndarray], np.ndarray, np.ndarray]:
    raw = f.metadata.get("lance:ivf")
    if raw is None:
        raise LanceFormatError(f"{f.path}: schema metadata 'lance:ivf' is missing")
    ivf = pb_fields(f.global_buffer(int(raw.decode())))
    offsets = np.asarray(pb_repeated_ints(ivf.get(2, [])), np.uint64)
    lengths = np.asarray(pb_repeated_ints(ivf.get(3, [])), np.uint64)
    cent = _tensor_f32(ivf[4][0], f"{f.path}: IVF centroids") if 4 in ivf else None
    if offsets.shape != lengths.shape:
        raise LanceFormatError(f"{f.path}: IVF offsets / lengths disagree")
    return cent, offsets, lengths


def read_ivf_pq_index(index_dir: str):
    """``_indices/<uuid>/`` -> ``IvfPqIndexData`` (centroids, codebook [m][256][dsub], partition offsets, row-major
    codes in partition order, row ids).  Raw vectors are not part of an index: pass them separately for refine."""
    from .index import IvfPqIndexData
    idx = LanceFile(os.path.join(index_dir, "index.idx"))
    aux = LanceFile(os.path.join(index_dir, "auxiliary.idx"))
    meta = idx.meta_json("lance:index")
    if str(meta.get("type", "")).upper() != "IVF_PQ":
        raise LanceFormatError(f"{index_dir}: index type {meta.get('type')!r} is not IVF_PQ")
    metric = {"l2": "l2", "euclidean": "l2", "cosine": "cosine", "dot": "dot"}.get(str(meta.get("distance_type", "l2")).lower())
    if metric is None:
        raise LanceFormatError(f"{index_dir}: distance type {meta.get('distance_type')!r} is not handled")
    cent, _, _ = _ivf_model(idx)
    if cent is None or cent.ndim != 2:
        raise LanceFormatError(f"{index_dir}: index.idx holds no centroid tensor")
    nlist, dim = cent.shape
    _, offsets, lengths = _ivf_model(aux)
    if offsets.shape[0] != nlist:
        raise LanceFormatError(f"{index_dir}: {offsets.shape[0]} partitions in auxiliary.idx, {nlist} centroids")
    sm = aux.meta_json("storage_metadata")
    pq = json.loads(sm[0]) if isinstance(sm, list) and sm and isinstance(sm[0], str) else (sm[0] if isinstance(sm, list) else sm)
    m, nbits = int(pq["num_sub_vectors"]), int(pq.get("nbits", 8))
    if nbits != 8:
        raise LanceFormatError(f"{index_dir}: {nbits}-bit PQ is not handled (SURVEY.md 8a: 8-bit codes)")
    if int(pq.get("dimension", dim)) != dim or dim % m:
        raise LanceFormatError(f"{index_dir}: PQ dimension {pq.get('dimension')} / m {m} do not match centroids of dim {dim}")
    dsub = dim // m
    cb = _tensor_f32(aux.global_buffer(int(pq["codebook_position"])), f"{index_dir}: PQ codebook")
    if cb.shape != (256, dim):
        raise LanceFormatError(f"{index_dir}: codebook tensor of shape {cb.shape}, expected (256, {dim})")
    codebook = np.ascontiguousarray(cb.reshape(256, m, dsub).transpose(1, 0, 2))          # [m][256][dsub]
    row_ids = aux.read_flat_column("_rowid", np.uint64)
    codes = aux.read_flat_column("__pq_code", np.uint8, m)
    n = row_ids.shape[0]
    if np.any(offsets + lengths > n) or int(lengths.sum()) != n:
        raise LanceFormatError(f"{index_dir}: partition lengths do not cover the {n} stored rows")
    order = np.argsort(offsets, kind="stable")
    if not np.array_equal(offsets[order][1:], (offsets[order] + lengths[order])[:-1]) or (n and offsets[order][0] != 0):
        raise LanceFormatError(f"{index_dir}: partitions are not contiguous in auxiliary.idx")
    part_off = np.zeros(nlist + 1, np.uint64)
    part_off[1:] = np.cumsum(lengths)
    # IvfPqIndexData keeps the codes partition-transposed ([m][n_p] per partition, SURVEY.md 8a row a6) -- the layout a
    # `transposed` file already has: the n_p * m bytes of a partition's file rows ARE its [m][n_p] matrix.  A
    # row-major file is transposed here.  Partitions are emitted in id order whatever their order in the file.
    transposed = bool(pq.get("transposed", False))
    codes_t = np.empty(n * m, np.uint8)
    ids = np.empty(n, np.uint64)
    for p in range(nlist):
        s, e = int(offsets[p]), int(offsets[p] + lengths[p])
        a, b = int(part_off[p]), int(part_off[p + 1])
        blk = codes[s:e]
        codes_t[a * m:b * m] = blk.reshape(-1) if transposed else np.ascontiguousarray(blk.T).reshape(-1)
        ids[a:b] = row_ids[s:e]
    return IvfPqIndexData(dim, nlist, m, metric, cent, codebook, part_off, codes_t, ids, None)


def find_index_dirs(table_uri: str) -> List[str]:
    """``<table>.lance/_indices/*`` directories that hold an IVF_PQ pair of files."""
    root = os.path.join(table_uri, "_indices")
    if not os.path.isdir(root):
        return []
    return [os.path.join(root, d) for d in sorted(os.listdir(root))
            if os.path.isfile(os.path.join(root, d, "index.idx")) and os.path.isfile(os.path.join(root, d, "auxiliary.idx"))]


# ------------------------------------------------------------------------------------------ writer (test fixtures only)
def _flat_encoding(bits: int) -> bytes:
    return pb_bytes(1, pb_int(1, bits) + pb_bytes(2, pb_int(1, 0) + pb_int(2, 0)))


def _page_encoding(array_encoding: bytes) -> bytes:
    any_msg = pb_bytes(1, ("type.googleapis.com" + ANY_ARRAY_ENCODING).encode()) + pb_bytes(2, array_encoding)
    return pb_bytes(2, pb_bytes(1, any_msg))                   # Encoding{direct{encoding}}


class _FileWriter:
    def __init__(self):
        self.buf = bytearray()
        self.col_meta: List[bytes] = []
        self.globals: List[Tuple[int, int]] = []
        self.fields: List[bytes] = []
        self.meta: Dict[str, bytes] = {}
        self.rows = 0

    def _append(self, b: bytes) -> Tuple[int, int]:
        while len(self.buf) % 64:
            self.buf.append(0)
        pos = len(self.buf)
        self.buf += b
        return pos, len(b)

    def add_column(self, name: str, logical_type: str, arr: np.ndarray, array_encoding: bytes, page_rows: int = 0):
        nrows = arr.shape[0]
        self.rows = nrows
        step = page_rows or max(nrows, 1)
        pages = b""
        for s in range(0, max(nrows, 1), step):
            part = np.ascontiguousarray(arr[s:s + step])
            pos, size = self._append(part.tobytes())
            pages += pb_bytes(2, pb_packed(1, [pos]) + pb_packed(2, [size]) + pb_int(3, part.shape[0]) +
                              pb_bytes(4, _page_encoding(array_encoding)))
        self.col_meta.append(pages)
        self.fields.append(pb_int(1, 2) + pb_bytes(2, name.encode()) + pb_int(3, len(self.fields)) +
                           pb_bytes(5, logical_type.encode()))

    def add_global(self, b: bytes) -> int:
        self.globals.append(self._append(b))
        return len(self.globals)                               # buffer 0 is the schema, written last

    def finish(self, path: str):
        schema = b"".join(pb_bytes(1, f) for f in self.fields)
        for k, v in self.meta.items():
            schema += pb_bytes(5, pb_bytes(1, k.encode()) + pb_bytes(2, v))
        gb0 = self._append(pb_bytes(1, schema) + pb_int(2, self.rows))
        col_meta_start = len(self.buf)
        cols = [self._append(c) for c in self.col_meta]
        if cols:
            col_meta_start = cols[0][0]
        cmo = len(self.buf)
        for pos, size in cols:
            self.buf += struct.pack("<QQ", pos, size)
        gbo = len(self.buf)
        for pos, size in [gb0] + self.globals:
            self.buf += struct.pack("<QQ", pos, size)
        self.buf += struct.pack("<QQQIIHH", col_meta_start, cmo, gbo, 1 + len(self.globals), len(cols), 2, 0) + MAGIC
        with open(path, "wb") as f:
            f.write(self.buf)


def _tensor_pb(a: np.ndarray) -> bytes:
    a = np.ascontiguousarray(a, np.float32)
    return pb_int(1, TENSOR_F32) + pb_packed(2, a.shape) + pb_bytes(3, a.tobytes())


def write_ivf_pq_index(index_dir: str, ix, transposed: bool = True, page_rows: int = 0) -> None:
    """Emit ``index.idx`` + ``auxiliary.idx`` for an ``IvfPqIndexData`` in the recalled layout (module docstring)."""
    os.makedirs(index_dir, exist_ok=True)
    nlist, m, dim = ix.nlist, ix.m, ix.dim
    off = np.asarray(ix.part_offsets, np.uint64)
    lengths = (off[1:] - off[:-1]).astype(np.uint64)
    ivf_aux = pb_packed(2, off[:-1]) + pb_packed(3, lengths)
    w = _FileWriter()
    g = w.add_global(ivf_aux + pb_bytes(4, _tensor_pb(ix.centroids.reshape(nlist, dim))))
    w.meta["lance:ivf"] = str(g).encode()
    w.meta["lance:index"] = json.dumps({"type": "IVF_PQ", "distance_type": ix.metric}).encode()
    w.finish(os.path.join(index_dir, "index.idx"))
    codes = np.empty((ix.nrows, m), np.uint8)
    for p in range(nlist):
        s, e = int(off[p]), int(off[p + 1])
        blk = np.asarray(ix.codes_t[s * m:e * m], np.uint8)              # the partition's [m][n_p] matrix
        codes[s:e] = blk.reshape(e - s, m) if transposed else np.ascontiguousarray(blk.reshape(m, e - s).T)
    a = _FileWriter()
    a.add_column("_rowid", "uint64", np.asarray(ix.row_ids, np.uint64), pb_bytes(2, pb_bytes(1, pb_bytes(1, _flat_encoding(64)))), page_rows)
    a.add_column("__pq_code", f"fixed_size_list:uint8:{m}", codes,
                 pb_bytes(3, pb_int(1, m) + pb_bytes(2, _flat_encoding(8))), page_rows)
    dsub = dim // m
    cb = np.ascontiguousarray(np.asarray(ix.codebook, np.float32).reshape(m, 256, dsub).transpose(1, 0, 2)).reshape(256, dim)
    gcb = a.add_global(_tensor_pb(cb))
    givf = a.add_global(ivf_aux)
    a.meta["lance:ivf"] = str(givf).encode()
    a.meta["storage_metadata"] = json.dumps([json.dumps({"codebook_position": gcb, "nbits": 8, "num_sub_vectors": m,
                                                         "dimension": dim, "transposed": bool(transposed)})]).encode()
    a.finish(os.path.join(index_dir, "auxiliary.idx"))
