"""chunk.Column / chunk.Chunk in the reference's exact memory layout, on numpy buffers.

Mirrors pkg/util/chunk/column.go:74-82 (Column{length, nullBitmap, offsets, data}) and
pkg/util/chunk/chunk.go:35-54 (Chunk{columns, sel, ...}): fixed-width little-endian `data`,
LSB-first `nullBitmap` where bit 1 means NOT NULL, optional selection vector `sel`.
Fixed-width columns and var-length string columns (int64 `offsets`, uint8 `data`) are modelled.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import abi


DECIMAL_CELL = 40   # bytes of one MyDecimal cell in a chunk column
DECIMAL_DTYPE = np.dtype((np.uint8, DECIMAL_CELL))   # numpy allocates it as (n, 40) uint8
VARLEN = -1         # elem_len of a var-length column (getFixedLen, codec.go:165)


def pack_not_null_bitmap(nulls: np.ndarray) -> np.ndarray:
    """bool array (True = NULL) -> Column.nullBitmap bytes (bit 1 = NOT NULL, LSB first)."""
    return np.packbits(~np.asarray(nulls, dtype=bool), bitorder="little")


def unpack_nulls(bitmap: np.ndarray, n: int) -> np.ndarray:
    """Column.nullBitmap bytes -> bool array (True = NULL) of length n."""
    bits = np.unpackbits(np.asarray(bitmap, dtype=np.uint8), bitorder="little")[:n]
    return bits == 0


class Column:
    """One chunk.Column.  Fixed width: `data` is a 1-D numpy array of int64/uint64/float64/float32, or an (n, 40) uint8
    array of MyDecimal cells (a DECIMAL column: types/mydecimal.go:236, copied whole into the column, column.go:41).
    Var-length (a string column, `offsets` given): `offsets` holds length + 1 int64 values and row r is the bytes
    data[offsets[r]:offsets[r + 1]] of the uint8 `data` (Column.GetString, column.go:715); elem_len is -1."""

    def __init__(self, data: np.ndarray, nulls: Optional[np.ndarray] = None, offsets: Optional[np.ndarray] = None):
        self.offsets: Optional[np.ndarray] = None
        if offsets is not None:
            self.offsets = np.ascontiguousarray(offsets, dtype=np.int64)
            data = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
            self.elem_len = VARLEN
        else:
            data = np.ascontiguousarray(data)
            if data.ndim == 2 and data.dtype == np.uint8 and data.shape[1] == DECIMAL_CELL:
                self.elem_len = DECIMAL_CELL
            elif data.dtype.itemsize in (4, 8):
                self.elem_len = int(data.dtype.itemsize)
            else:
                raise ValueError("only 4/8-byte fixed-width columns, 40-byte DECIMAL cells and var-length columns are modelled")
        self.data = data
        self.length = int(data.shape[0]) if offsets is None else int(self.offsets.shape[0]) - 1
        if nulls is not None:
            nulls = np.asarray(nulls, dtype=bool)
            if nulls.shape[0] != self.length:
                raise ValueError("nulls length mismatch")
            self.null_bitmap: Optional[np.ndarray] = pack_not_null_bitmap(nulls)
        else:
            self.null_bitmap = None

    @classmethod
    def strings(cls, values: Sequence[Optional[bytes]]) -> "Column":
        """A var-length column of the given rows; None is NULL (an empty row under the bitmap)."""
        lens = np.array([0 if v is None else len(v) for v in values], dtype=np.int64)
        offsets = np.zeros(len(values) + 1, dtype=np.int64)
        np.cumsum(lens, out=offsets[1:])
        data = np.frombuffer(b"".join(b"" if v is None else bytes(v) for v in values), dtype=np.uint8).copy()
        nulls = np.array([v is None for v in values], dtype=bool)
        return cls(data, nulls if nulls.any() else None, offsets)

    @property
    def is_varlen(self) -> bool:
        return self.offsets is not None

    def get_bytes(self, i: int) -> bytes:
        """Column.GetString: the bytes of row i of a var-length column"""
        return self.data[self.offsets[i]:self.offsets[i + 1]].tobytes()

    def values(self) -> list:
        """the rows of a var-length column as bytes, None where NULL"""
        nl = self.nulls()
        return [None if nl[i] else self.get_bytes(i) for i in range(self.length)]

    def take(self, idx: np.ndarray) -> "Column":
        """rows idx (int array) of the column, in that order, as a new dense column (the gather of a sel vector)"""
        idx = np.asarray(idx, dtype=np.int64)
        nl = self.nulls()[idx] if self.null_bitmap is not None else None
        if nl is not None and not nl.any():
            nl = None
        if not self.is_varlen:
            return Column(self.data[idx], nl)
        starts, ends = self.offsets[idx], self.offsets[idx + 1]
        offsets = np.zeros(len(idx) + 1, dtype=np.int64)
        np.cumsum(ends - starts, out=offsets[1:])
        pos = np.repeat(starts - offsets[:-1], ends - starts) + np.arange(int(offsets[-1]), dtype=np.int64)
        return Column(self.data[pos], nl, offsets)

    # Column.IsNull column.go:225
    def is_null(self, i: int) -> bool:
        if self.null_bitmap is None:
            return False
        return ((int(self.null_bitmap[i >> 3]) >> (i & 7)) & 1) == 0

    def nulls(self) -> np.ndarray:
        if self.null_bitmap is None:
            return np.zeros(self.length, dtype=bool)
        return unpack_nulls(self.null_bitmap, self.length)

    def to_struct(self) -> abi.TgColumn:
        s = abi.TgColumn()
        s.length = self.length
        s.null_bitmap = self.null_bitmap.ctypes.data if self.null_bitmap is not None else None
        s.offsets = self.offsets.ctypes.data if self.is_varlen else None
        s.data = self.data.ctypes.data if (self.data.size if self.is_varlen else self.length) else None
        s.elem_len = self.elem_len
        return s

    def slice(self, lo: int, hi: int) -> "Column":
        nl = self.nulls()[lo:hi] if self.null_bitmap is not None else None
        if self.is_varlen:
            o = self.offsets[lo:hi + 1]
            return Column(self.data[o[0]:o[-1]].copy(), nl, o - o[0])
        return Column(self.data[lo:hi].copy(), nl)


def concat_columns(cols: Sequence[Column]) -> Column:
    """the rows of several columns of one type, one after the other, as one dense column (sel vectors not applied)"""
    nl = np.concatenate([c.nulls() for c in cols]) if any(c.null_bitmap is not None for c in cols) else None
    if nl is not None and not nl.any():
        nl = None
    if not cols[0].is_varlen:
        return Column(np.concatenate([c.data for c in cols]), nl)
    offsets, data, at = [np.zeros(1, dtype=np.int64)], [], 0
    for c in cols:
        offsets.append(c.offsets[1:] - c.offsets[0] + at)
        data.append(c.data[c.offsets[0]:c.offsets[-1]])
        at += int(c.offsets[-1] - c.offsets[0])
    return Column(np.concatenate(data) if data else np.zeros(0, np.uint8), nl, np.concatenate(offsets))


class Chunk:
    """chunk.Chunk: columns + optional sel (logical row i -> physical row sel[i])."""

    def __init__(self, columns: Sequence[Column], sel: Optional[np.ndarray] = None):
        self.columns: List[Column] = list(columns)
        self.sel = None if sel is None else np.ascontiguousarray(sel, dtype=np.int64)
        self._keep = None

    # Chunk.NumRows chunk.go:384
    def num_rows(self) -> int:
        if self.sel is not None:
            return int(self.sel.shape[0])
        return self.columns[0].length if self.columns else 0

    def num_cols(self) -> int:
        return len(self.columns)

    def to_struct(self) -> abi.TgChunk:
        n = len(self.columns)
        arr = (abi.TgColumn * max(n, 1))()
        for i, c in enumerate(self.columns):
            arr[i] = c.to_struct()
        s = abi.TgChunk()
        s.ncols = n
        s.cols = C.cast(arr, C.POINTER(abi.TgColumn))
        s.sel = self.sel.ctypes.data if self.sel is not None else None
        s.nsel = self.num_rows() if self.sel is not None else 0
        self._keep = arr
        return s

    def split(self, max_rows: int) -> List["Chunk"]:
        """Cut into chunks of at most max_rows physical rows (tidb_max_chunk_size = 1024)."""
        assert self.sel is None
        n = self.num_rows()
        out = []
        for lo in range(0, n, max_rows):
            hi = min(n, lo + max_rows)
            out.append(Chunk([c.slice(lo, hi) for c in self.columns]))
        return out


def chunk_array(chunks: Sequence[Chunk]):
    """C array of tg_chunk for a list of chunks (keeps the backing structs alive on the result)."""
    arr = (abi.TgChunk * max(len(chunks), 1))()
    for i, c in enumerate(chunks):
        arr[i] = c.to_struct()
    arr._chunks = list(chunks)  # keep alive
    return arr


class MutChunk:
    """Caller-owned output chunk (tg_mut_chunk): numpy buffers the library fills.  A var-length column (elem_len -1) has
    capacity + 1 int64 offsets and `data_cap` bytes, described to the library by `varlen` (one tg_mut_varlen per
    column, zeros for the fixed-width ones)."""

    def __init__(self, elem_lens: Sequence[int], capacity_rows: int, dtypes: Optional[Sequence] = None, data_cap: int = 0):
        self.capacity = int(capacity_rows)
        self.elem_lens = list(elem_lens)
        self.data = []
        self.bitmaps = []
        self.offsets: List[Optional[np.ndarray]] = []
        self.varlen = (abi.TgMutVarlen * max(len(elem_lens), 1))()
        for i, el in enumerate(elem_lens):
            if el == VARLEN:
                self.data.append(np.zeros(max(int(data_cap), 1), dtype=np.uint8))
                self.offsets.append(np.zeros(max(self.capacity, 1) + 1, dtype=np.int64))
                self.varlen[i].offsets = self.offsets[i].ctypes.data
                self.varlen[i].data = self.data[i].ctypes.data
                self.varlen[i].data_cap = int(data_cap)
            else:
                dt = dtypes[i] if dtypes is not None else (np.int64 if el == 8 else np.float32)
                self.data.append(np.zeros(max(self.capacity, 1), dtype=dt))
                self.offsets.append(None)
            self.bitmaps.append(np.zeros((max(self.capacity, 1) + 7) // 8, dtype=np.uint8))
        self._cols = (abi.TgMutColumn * max(len(elem_lens), 1))()
        for i, el in enumerate(elem_lens):
            self._cols[i].null_bitmap = self.bitmaps[i].ctypes.data
            self._cols[i].data = self.data[i].ctypes.data
            self._cols[i].elem_len = el
        self.struct = abi.TgMutChunk()
        self.struct.ncols = len(elem_lens)
        self.struct.cols = C.cast(self._cols, C.POINTER(abi.TgMutColumn))
        self.struct.capacity_rows = self.capacity

    def columns(self, nrows: int):
        """-> list of (values ndarray[:nrows], nulls bool ndarray[:nrows]); a var-length column's values are its rows as
        bytes (None where NULL) in an object array"""
        out = []
        for i, (d, b) in enumerate(zip(self.data, self.bitmaps)):
            nl = unpack_nulls(b, nrows)
            if self.offsets[i] is None:
                out.append((d[:nrows].copy(), nl))
            else:
                o = self.offsets[i]
                out.append((np.array([None if nl[r] else d[o[r]:o[r + 1]].tobytes() for r in range(nrows)], dtype=object), nl))
        return out

    def column(self, i: int, nrows: int) -> Column:
        """output column i of the first nrows rows as a Column (var-length columns keep their offsets)"""
        nl = unpack_nulls(self.bitmaps[i], nrows)
        nl = nl if nl.any() else None
        if self.offsets[i] is None:
            return Column(self.data[i][:nrows].copy(), nl)
        o = self.offsets[i][:nrows + 1].copy()
        return Column(self.data[i][:o[-1]].copy(), nl, o)
