"""Replay-ring files: one uncompressed zip64 `.npz`, streamed through two bounded host buffers.

Layout (DESIGN.md §2): a `meta` member first (0-d unicode array holding JSON: format version, ring class, capacity, cameras,
frame shape, T / S / A and the host bookkeeping), then one `.npy` member per ring field over the filled slots `[0, n)`:
`frames/<cam>` (n, H, W, C) u8, `state`, `next_state`, `actions`, `rewards`, `masks`, `dones`, `valid`.  `np.load` opens the
file; the zip CRC-32 of each member is the integrity check.

The writer and reader here are host-side and device-agnostic: they move bytes between the file and a `Stager`, which owns
two staging buffers of `chunk_bytes` each and copies chunks between them and the arrays.  `HostStager` does that with numpy
arrays (tests, tools); the ring's CUDA stager (replay_buffer.py) does it with pinned buffers and async copies, so the copy of
chunk i + 1 overlaps the file I/O of chunk i and host memory stays at two chunks whatever the ring size.
"""
from __future__ import annotations

import io
import json
import os
import zipfile
from typing import List, Sequence, Tuple

import numpy as np

FORMAT_VERSION = 1
CHUNK_BYTES = 32 << 20          # per staging buffer; a save or load holds two (a power of two: no rounding in torch's pinned pool)


class Field:
    """One array of the file: `name` (member name without `.npy`), its dtype and shape, and `src` - whatever the stager
    copies from (save) or into (load): a numpy array for `HostStager`, a flat u8 device tensor for the CUDA stager."""

    def __init__(self, name: str, dtype, shape: Sequence[int], src):
        self.name, self.dtype, self.shape, self.src = name, np.dtype(dtype), tuple(int(s) for s in shape), src

    @property
    def nbytes(self) -> int:
        return int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize


class HostStager:
    """`Stager` over numpy arrays: copies are immediate memcpys through two bytearrays of `chunk_bytes`."""

    def __init__(self, chunk_bytes: int = CHUNK_BYTES):
        self.chunk_bytes = int(chunk_bytes)
        self._buf = [np.empty(self.chunk_bytes, np.uint8) for _ in range(2)]
        self._len = [0, 0]

    @staticmethod
    def _bytes(a: np.ndarray) -> np.ndarray:
        return a.reshape(-1).view(np.uint8)

    def d2h(self, k: int, src, lo: int, hi: int):          # start copying bytes [lo, hi) of src into buffer k
        self._buf[k][:hi - lo] = self._bytes(src)[lo:hi]
        self._len[k] = hi - lo

    def wait(self, k: int) -> memoryview:                   # buffer k once its d2h is complete
        return memoryview(self._buf[k][:self._len[k]])

    def host(self, k: int, n: int) -> memoryview:           # buffer k, writable, once its previous h2d is complete
        return memoryview(self._buf[k][:n])

    def h2d(self, k: int, dst, lo: int, hi: int):           # start copying the first hi - lo bytes of buffer k to dst[lo, hi)
        self._bytes(dst)[lo:hi] = self._buf[k][:hi - lo]

    def finish(self):
        pass


def _chunks(fields: Sequence[Field], chunk: int) -> List[Tuple[int, int, int]]:
    return [(i, lo, min(lo + chunk, f.nbytes)) for i, f in enumerate(fields) for lo in range(0, f.nbytes, chunk)]


def _npy_header(dtype: np.dtype, shape) -> bytes:
    b = io.BytesIO()
    np.lib.format.write_array_header_1_0(b, {"descr": np.lib.format.dtype_to_descr(dtype), "fortran_order": False,
                                            "shape": tuple(shape)})
    return b.getvalue()


def _zinfo(name: str) -> zipfile.ZipInfo:
    zi = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
    zi.compress_type = zipfile.ZIP_STORED
    return zi


def write_ring_file(path, meta: dict, fields: Sequence[Field], stager) -> int:
    """Writes `meta` and `fields` to `path` atomically (into `path + ".tmp"`, then `os.replace`); returns the file's size.
    On any error the temporary file is removed and an existing `path` is left as it was."""
    path = os.fspath(path)
    tmp = path + ".tmp"
    chunks = _chunks(fields, stager.chunk_bytes)
    try:
        with open(tmp, "wb") as fp:
            with zipfile.ZipFile(fp, "w", compression=zipfile.ZIP_STORED, allowZip64=True) as zf:
                with zf.open(_zinfo("meta"), "w", force_zip64=True) as m:
                    text = np.array(json.dumps(meta, sort_keys=True))
                    m.write(_npy_header(text.dtype, ()))
                    m.write(text.tobytes())
                if chunks:
                    fi, lo, hi = chunks[0]
                    stager.d2h(0, fields[fi].src, lo, hi)
                ci = 0
                for fi, f in enumerate(fields):
                    with zf.open(_zinfo(f.name), "w", force_zip64=True) as m:
                        m.write(_npy_header(f.dtype, f.shape))
                        while ci < len(chunks) and chunks[ci][0] == fi:
                            if ci + 1 < len(chunks):             # its buffer's previous chunk (ci - 1) is already in the file
                                nf, lo, hi = chunks[ci + 1]
                                stager.d2h((ci + 1) & 1, fields[nf].src, lo, hi)
                            m.write(stager.wait(ci & 1))
                            ci += 1
            fp.flush()
            os.fsync(fp.fileno())                                # the new file is on disk before it replaces the old one
        stager.finish()
        os.replace(tmp, path)
    except BaseException:
        stager.finish()
        try:
            os.remove(tmp)
        except OSError:
            pass
        raise
    return os.path.getsize(path)


_DAMAGE = (zipfile.BadZipFile, EOFError, KeyError, ValueError)     # what zipfile / numpy raise on a damaged archive or member


def _corrupt(path, what, err) -> ValueError:
    return ValueError(f"replay file {path!r}: {what}: {err}")


def read_meta(path) -> dict:
    """The `meta` member of a ring file (ValueError if the file is not one, or is damaged)."""
    path = os.fspath(path)
    try:
        zf = zipfile.ZipFile(path, "r")
    except _DAMAGE as e:
        raise _corrupt(path, "not a complete zip archive", e) from e
    try:
        with zf, zf.open("meta.npy") as m:
            arr = np.lib.format.read_array(m, allow_pickle=False)
            if m.read(1):
                raise ValueError("member is longer than its header says")
        return json.loads(str(arr[()]))
    except _DAMAGE as e:
        raise _corrupt(path, "meta", e) from e


def check_meta(saved: dict, expected: dict):
    """ValueError naming the first field where a file's meta and the receiving ring disagree."""
    for key in ("version", "class", "capacity", "cams", "frame_shape", "T", "S", "A"):
        got, want = saved.get(key), expected[key]
        if got != (list(want) if isinstance(want, tuple) else want):
            raise ValueError(f"replay file does not fit this buffer: {key} is {got!r} in the file, {want!r} here")


def read_ring_file(path, fields: Sequence[Field], stager):
    """Streams the members named by `fields` (whose dtypes and shapes must match the file's headers) into their `src`.
    Raises ValueError naming the member on a header mismatch, a short member or a CRC error; the CRC of a member is checked
    when its last byte is read, after earlier chunks were already copied out, so a caller must discard what it loaded on error."""
    path = os.fspath(path)
    chunk = stager.chunk_bytes
    k = 0
    try:
        zf = zipfile.ZipFile(path, "r")
    except _DAMAGE as e:
        raise _corrupt(path, "not a complete zip archive", e) from e
    try:
        with zf:
            for f in fields:
                try:
                    with zf.open(f.name + ".npy") as m:
                        version = np.lib.format.read_magic(m)
                        read_hdr = np.lib.format.read_array_header_1_0 if version == (1, 0) else np.lib.format.read_array_header_2_0
                        shape, fortran, dtype = read_hdr(m)
                        if tuple(shape) != f.shape or np.dtype(dtype) != f.dtype or fortran:
                            raise ValueError(f"file holds {np.dtype(dtype)}{tuple(shape)}, this buffer expects {f.dtype}{f.shape}")
                        for lo in range(0, f.nbytes, chunk):
                            hi = min(lo + chunk, f.nbytes)
                            got = m.readinto(stager.host(k, hi - lo))
                            if got != hi - lo:
                                raise ValueError(f"member ends after {lo + got} of {f.nbytes} bytes")
                            stager.h2d(k, f.src, lo, hi)
                            k ^= 1
                        if m.read(1):
                            raise ValueError("member is longer than its header says")
                except _DAMAGE as e:
                    raise _corrupt(path, f.name, "member missing" if isinstance(e, KeyError) else e) from e
    finally:
        stager.finish()
