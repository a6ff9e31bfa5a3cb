"""CPU: the replay-file writer / reader (serl_b200/data/replay_io.py) over numpy arrays - streaming in chunks smaller than the
arrays, the standard .npz layout, CRC and truncation detection, meta validation, atomic replacement."""
import json
import os
import zipfile

import numpy as np
import pytest

from serl_b200.data import replay_io as RIO

CHUNK = 4096


def _arrays(n=300, seed=0):
    rng = np.random.default_rng(seed)
    return {"frames/front": rng.integers(0, 256, (n, 12, 12, 3), dtype=np.uint8),      # 129 600 B: 32 chunks
            "state": rng.standard_normal((n, 7)).astype(np.float32),
            "actions": rng.uniform(-1, 1, (n, 4)).astype(np.float32),
            "rewards": rng.random(n).astype(np.float32),
            "dones": (rng.random(n) < 0.1).astype(np.uint8),
            "valid": (rng.random(n) < 0.9).astype(np.uint8)}


def _meta(**kw):
    m = {"version": RIO.FORMAT_VERSION, "class": "MemoryEfficientReplayBuffer", "capacity": 400, "cams": ["front"],
         "frame_shape": [12, 12, 3], "T": 1, "S": 7, "A": 4, "_size": 300, "_insert_index": 300, "_seed": 5, "_draw_step": 3}
    m.update(kw)
    return m


def _fields(arrays):
    return [RIO.Field(k, a.dtype, a.shape, a) for k, a in arrays.items()]


def _save(path, arrays, meta=None):
    return RIO.write_ring_file(path, meta or _meta(), _fields(arrays), RIO.HostStager(CHUNK))


def _empty_like(arrays):
    return {k: np.full_like(a, 7) for k, a in arrays.items()}


def test_round_trip_larger_than_chunk(tmp_path):
    arrays = _arrays()
    assert arrays["frames/front"].nbytes > 10 * CHUNK
    p = tmp_path / "ring.npz"
    size = _save(p, arrays)
    assert size == os.path.getsize(p) and not os.path.exists(str(p) + ".tmp")
    assert RIO.read_meta(p) == _meta()
    out = _empty_like(arrays)
    RIO.read_ring_file(p, _fields(out), RIO.HostStager(CHUNK))
    for k in arrays:
        np.testing.assert_array_equal(out[k], arrays[k])


def test_chunk_boundaries_and_empty_members(tmp_path):
    """Sizes at, around and below the chunk size, and a zero-row member (an empty ring)."""
    arrays = {"a": np.arange(CHUNK, dtype=np.uint8).reshape(CHUNK, 1), "b": np.arange(CHUNK + 1, dtype=np.uint8),
              "c": np.arange(3 * CHUNK // 4 - 1, dtype=np.float32), "d": np.zeros((0, 5, 5, 3), np.uint8), "e": np.ones(1, np.uint8)}
    p = tmp_path / "ring.npz"
    _save(p, arrays)
    out = _empty_like(arrays)
    RIO.read_ring_file(p, _fields(out), RIO.HostStager(CHUNK))
    for k in arrays:
        np.testing.assert_array_equal(out[k], arrays[k])


def test_np_load_reads_the_file(tmp_path):
    arrays = _arrays(n=50)
    p = tmp_path / "ring.npz"
    _save(p, arrays)
    with np.load(p) as z:
        assert set(z.files) == {"meta", *arrays}
        assert json.loads(str(z["meta"])) == _meta()
        for k, a in arrays.items():
            assert z[k].dtype == a.dtype
            np.testing.assert_array_equal(z[k], a)
    with zipfile.ZipFile(p) as zf:                      # standard, uncompressed, CRC'd members
        assert zf.testzip() is None
        assert all(i.compress_type == zipfile.ZIP_STORED for i in zf.infolist())
        assert zf.namelist()[0] == "meta.npy"


@pytest.mark.parametrize("member", ["frames/front.npy", "valid.npy", "meta.npy"])
def test_flipped_byte_is_rejected(tmp_path, member):
    arrays = _arrays()
    p = tmp_path / "ring.npz"
    _save(p, arrays)
    raw = bytearray(p.read_bytes())
    with zipfile.ZipFile(p) as zf:
        info = zf.getinfo(member)
    # the member's data follows its local header: 30 bytes, then the name and the extra field (lengths at bytes 26 and 28)
    off = info.header_offset
    name_len, extra_len = (int.from_bytes(raw[off + i:off + i + 2], "little") for i in (26, 28))
    raw[off + 30 + name_len + extra_len + info.file_size // 2] ^= 0x40
    p.write_bytes(bytes(raw))
    with pytest.raises(ValueError, match=member.replace(".npy", "")):
        if member == "meta.npy":
            RIO.read_meta(p)
        else:
            RIO.read_ring_file(p, _fields(_empty_like(arrays)), RIO.HostStager(CHUNK))


@pytest.mark.parametrize("keep", [0.999, 0.5, 0.01])
def test_truncated_file_is_rejected(tmp_path, keep):
    arrays = _arrays()
    p = tmp_path / "ring.npz"
    _save(p, arrays)
    raw = p.read_bytes()
    p.write_bytes(raw[:int(len(raw) * keep)])
    with pytest.raises(ValueError, match="ring.npz"):
        RIO.read_meta(p)
    with pytest.raises(ValueError, match="ring.npz"):
        RIO.read_ring_file(p, _fields(_empty_like(arrays)), RIO.HostStager(CHUNK))


def test_member_shape_or_dtype_mismatch_names_the_field(tmp_path):
    arrays = _arrays()
    p = tmp_path / "ring.npz"
    _save(p, arrays)
    out = _empty_like(arrays)
    out["state"] = np.zeros((300, 8), np.float32)
    with pytest.raises(ValueError, match="state"):
        RIO.read_ring_file(p, _fields(out), RIO.HostStager(CHUNK))
    out = _empty_like(arrays)
    out["dones"] = np.zeros(300, np.float32)
    with pytest.raises(ValueError, match="dones"):
        RIO.read_ring_file(p, _fields(out), RIO.HostStager(CHUNK))
    out = _empty_like(arrays)
    out["masks"] = np.zeros(300, np.float32)
    with pytest.raises(ValueError, match="masks: member missing"):
        RIO.read_ring_file(p, _fields(out), RIO.HostStager(CHUNK))


@pytest.mark.parametrize("key,value", [("version", 99), ("class", "ReplayBuffer"), ("capacity", 401), ("cams", ["front", "wrist"]),
                                       ("frame_shape", [128, 128, 3]), ("T", 2), ("S", 8), ("A", 3)])
def test_meta_mismatch_names_the_field(key, value):
    want = {k: (tuple(v) if isinstance(v, list) else v) for k, v in _meta().items()}
    RIO.check_meta(_meta(), want)
    with pytest.raises(ValueError, match=rf"\b{key}\b"):
        RIO.check_meta(_meta(**{key: value}), want)


def test_failed_save_leaves_the_previous_file(tmp_path):
    arrays = _arrays()
    p = tmp_path / "ring.npz"
    _save(p, arrays)
    before = p.read_bytes()

    class Failing(RIO.HostStager):
        def d2h(self, k, src, lo, hi):
            if lo >= 8 * CHUNK:
                raise OSError("device copy failed")
            super().d2h(k, src, lo, hi)

    with pytest.raises(OSError, match="device copy failed"):
        RIO.write_ring_file(p, _meta(_size=1), _fields(_arrays(seed=1)), Failing(CHUNK))
    assert p.read_bytes() == before and not os.path.exists(str(p) + ".tmp")
    os.mkdir(str(p) + ".tmp")                              # the temporary cannot be created
    with pytest.raises(OSError):
        _save(p, _arrays(seed=2))
    assert p.read_bytes() == before
