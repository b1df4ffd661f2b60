"""The two cuts of a batch decode on the device, on every execute path.

1. Output chunks inside one call (run_decompress, zb_api.cu): a call whose output is copied back is cut by frame count
   into one chunk per 48 MiB of output (ZB200_OUT_CHUNK_BYTES replaces the 48 MiB), at most 32 and never more than
   there are frames; the copy of chunk k overlaps the kernels of chunk k + 1.
2. Sub-batches over pipeline contexts (ZstdDecompressor._run_contiguous): a BufferWithSegments of enough input is split
   into sub-batches of ~SUB_BATCH_INPUT_BYTES, run on PIPELINE_DEPTH contexts per device, each with its own arenas,
   pinned pool and copy of the dictionary; the lowest failing item wins, with its global index.

Frames are the reference's; outputs are compared with the source bytes, and with RefZstd.decompress on a sample."""
import ctypes as C

import numpy as np
import pytest
import torch

import corpus
import python_zstandard_b200 as zstd
from python_zstandard_b200 import _native
from oracle import have_ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason="oracle/_ref is built from /root/reference")]

MODES = {"lane-per-frame": ("0", None), "blocks+tiles": ("1", "0"), "blocks+pointer-jumping": ("1", "1"), "auto": (None, None)}


@pytest.fixture(params=list(MODES))
def mode(request, monkeypatch):
    for k, v in zip(("ZB200_BLOCK_PATH", "ZB200_CHASE"), MODES[request.param]):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, v)
    monkeypatch.delenv("ZB200_OUT_CHUNK_BYTES", raising=False)
    return request.param


@pytest.fixture
def auto(monkeypatch):
    for k in ("ZB200_BLOCK_PATH", "ZB200_CHASE", "ZB200_OUT_CHUNK_BYTES"):
        monkeypatch.delenv(k, raising=False)


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


def _table(lens):
    lens = np.asarray(lens, dtype=np.uint64)
    off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    return np.stack([off, lens], axis=1).astype(np.uint64)


def _text(n):
    """n bytes of text, the corpus repeated with a running counter every 4 KiB so no two stretches are equal."""
    t = corpus.text_corpus()
    reps = n // len(t) + 1
    out = np.tile(t, reps)[:n].copy()
    out[::4096] = (np.arange((n + 4095) // 4096) * 2654435761 >> 7).astype(np.uint8)
    return out


def _compress(ref, blob, lens, level=3, checksum=False, dct=b""):
    lens = np.asarray(lens, dtype=np.uint64)
    off = _table(lens)[:, 0].copy()
    cblob, clens = ref.batch(True, blob, off, lens, level=level, threads=8, checksum=checksum, dict_data=dct)
    return cblob, clens


def _bws(cblob, clens):
    return zstd.BufferWithSegments(cblob, _table(clens).tobytes())


def _sample(ref, out, cblob, clens, lens, blob, dct=b"", every=97):
    coff = _table(clens)[:, 0]; off = _table(lens)[:, 0]
    for i in range(0, len(lens), every):
        f = cblob[int(coff[i]):int(coff[i] + clens[i])].tobytes()
        want = blob[int(off[i]):int(off[i] + lens[i])].tobytes()
        assert out[i].tobytes() == ref.decompress(f, int(lens[i]), dct) == want, i


def _host_bytes(out):
    return b"".join(b.tobytes() for b in out._buffers)


K_ENTROPY, K_EXECUTE = 2, 3          # ZB200_K_ENTROPY, ZB200_K_EXECUTE (zb200.h): launch counts, kept with or without profiling


class _Launches:
    """What the last calls on the default context launched: run_decompress opens one EXECUTE span per output chunk, one
    ENTROPY span per chunk on the lane-per-frame path and a single one on the block path; zb200_last_chase_rounds is
    above 0 when the pointer-jumping stage ran.  (Batches that are not cut into sub-batches run on that context.)"""
    def __enter__(self):
        self.ctx = _native.Context.get(_native.default_device())
        self.ctx.L.zb200_profile_reset(self.ctx.h)
        return self

    def __exit__(self, *exc):
        ms, n = (C.c_float * _native.K_COUNT)(), (C.c_uint32 * _native.K_COUNT)()
        self.ctx.L.zb200_profile_read(self.ctx.h, ms, n)
        self.entropy, self.execute = int(n[K_ENTROPY]), int(n[K_EXECUTE])
        self.chase_rounds = int(self.ctx.L.zb200_last_chase_rounds(self.ctx.h))
        return False


# ---------------------------------------------------------------- the real chunk size, automatic path choice
def test_200_frames_of_1_mib_in_4_chunks_on_the_block_path(ref, auto):
    """200 MiB of output: four chunks of 50 frames; 1 MiB frames of eight blocks take the block path (zb_execute_big)."""
    lens = [1 << 20] * 200
    blob = _text(sum(lens))
    cblob, clens = _compress(ref, blob, lens, level=1, checksum=True)
    with _Launches() as k:
        out = zstd.ZstdDecompressor().multi_decompress_to_buffer(_bws(cblob, clens))
    assert (k.execute, k.entropy, k.chase_rounds) == (4, 1, 0)           # four chunks, block path, zb_execute_big
    assert np.array_equal(np.frombuffer(_host_bytes(out), dtype=np.uint8), blob)
    _sample(ref, out, cblob, clens, lens, blob, every=37)


def test_8_frames_of_16_mib_in_2_chunks_with_pointer_jumping(ref, auto):
    """128 MiB of output in two chunks of four frames: few frames of many blocks, the pointer-jumping stage over each
    chunk's output bytes."""
    lens = [16 << 20] * 8
    blob = _text(sum(lens))
    cblob, clens = _compress(ref, blob, lens, level=1)
    with _Launches() as k:
        out = zstd.ZstdDecompressor().multi_decompress_to_buffer(_bws(cblob, clens))
    assert (k.execute, k.entropy) == (2, 1) and k.chase_rounds > 0        # two chunks, block path, pointer jumping
    assert np.array_equal(np.frombuffer(_host_bytes(out), dtype=np.uint8), blob)
    _sample(ref, out, cblob, clens, lens, blob, every=3)


def test_32k_list_items_of_mixed_sizes_lane_per_frame(ref, auto):
    """~32 K list items of up to 4 KiB, with a 64 KiB item every 24th: ~150 MiB, three chunks of equal frame count whose
    output sizes differ; a lane per frame."""
    rng = np.random.default_rng(31)
    n = 32768
    lens = np.where(np.arange(n) % 24 == 5, 64 << 10, rng.integers(1, 4097, n)).astype(np.uint64)
    blob = _text(int(lens.sum()))
    cblob, clens = _compress(ref, blob, lens, level=3, checksum=True)
    coff = _table(clens)[:, 0]
    items = [cblob[int(o):int(o + l)].tobytes() for o, l in zip(coff, clens)]
    with _Launches() as k:
        out = zstd.ZstdDecompressor().multi_decompress_to_buffer(items)
    chunks = int(lens.sum()) // (48 << 20)
    assert chunks >= 2 and (k.execute, k.entropy, k.chase_rounds) == (chunks, chunks, 0)     # a lane per frame, per chunk
    assert len(out) == n
    assert np.array_equal(np.frombuffer(_host_bytes(out), dtype=np.uint8), blob)
    _sample(ref, out, cblob, clens, lens, blob, every=1013)


# ---------------------------------------------------------------- chunks forced small, every path
def _mixed_batch(ref, rng):
    """~24 MiB: 3000 small frames (1 B .. 4 KiB), 40 of 100 KiB and 6 of ~1.5 MiB, shuffled in runs so chunks differ."""
    lens = np.concatenate([rng.integers(1, 4097, 3000), [100 << 10] * 40, rng.integers(1 << 20, 2 << 20, 6)]).astype(np.uint64)
    order = np.argsort(rng.integers(0, 12, len(lens)), kind="stable")
    lens = lens[order]
    blob = _text(int(lens.sum()))
    cblob, clens = _compress(ref, blob, lens, level=3, checksum=True)
    return blob, lens, cblob, clens


@pytest.fixture(scope="module")
def mixed(ref):
    return _mixed_batch(ref, np.random.default_rng(41))


def test_32_chunks_on_every_path(ref, mode, mixed, monkeypatch):
    """A chunk size of 256 KiB asks for ~96 chunks: the cap of 32 binds."""
    blob, lens, cblob, clens = mixed
    monkeypatch.setenv("ZB200_OUT_CHUNK_BYTES", str(256 << 10))
    with _Launches() as k:
        out = zstd.ZstdDecompressor().multi_decompress_to_buffer(_bws(cblob, clens))
    assert k.execute == 32, mode
    assert np.array_equal(np.frombuffer(_host_bytes(out), dtype=np.uint8), blob), mode
    _sample(ref, out, cblob, clens, lens, blob, every=211)


def test_one_chunk_per_frame_on_every_path(ref, mode, monkeypatch):
    """Twelve frames of 64 B .. 3 MiB with a chunk size of 1 byte: clamped to one chunk per frame, empty ones included."""
    lens = np.array([3 << 20, 64, 0, 2 << 20, 5000, 1 << 20, 0, 0, 700000, 4096, 3 << 20, 1], dtype=np.uint64)
    blob = _text(int(lens.sum()))
    cblob, clens = _compress(ref, blob, lens, level=2, checksum=True)
    monkeypatch.setenv("ZB200_OUT_CHUNK_BYTES", "1")
    with _Launches() as k:
        out = zstd.ZstdDecompressor().multi_decompress_to_buffer(_bws(cblob, clens))
    assert k.execute == len(lens), mode
    assert np.array_equal(np.frombuffer(_host_bytes(out), dtype=np.uint8), blob), mode
    assert [len(out[i]) for i in range(len(lens))] == lens.tolist()
    _sample(ref, out, cblob, clens, lens, blob, every=1)


def test_damaged_frame_in_a_late_chunk(ref, mode, mixed, monkeypatch):
    """A wrong checksum in chunk 29 of 32 and a corrupt frame in chunk 31: the first is the one raised, with its index."""
    blob, lens, cblob, clens = mixed
    cblob = cblob.copy()
    coff = _table(clens)[:, 0]
    n = len(lens)
    wrong, corrupt = n * 29 // 32 + 1, n * 31 // 32 + 2
    cblob[int(coff[wrong] + clens[wrong]) - 1] ^= 0x5A                     # the content checksum's last byte
    cblob[int(coff[corrupt]) + 7: int(coff[corrupt] + clens[corrupt]) - 8] ^= 0x33
    monkeypatch.setenv("ZB200_OUT_CHUNK_BYTES", str(256 << 10))
    with pytest.raises(zstd.ZstdError, match=r"error decompressing item %d: Restored data doesn't match checksum" % wrong):
        zstd.ZstdDecompressor().multi_decompress_to_buffer(_bws(cblob, clens))


def test_device_call_equals_the_cut_host_call(mode, mixed, monkeypatch):
    """The same batch through DeviceBufferWithSegments (one call, one chunk) gives the bytes of the host call cut in 32."""
    blob, lens, cblob, clens = mixed
    monkeypatch.setenv("ZB200_OUT_CHUNK_BYTES", str(256 << 10))
    host = _host_bytes(zstd.ZstdDecompressor().multi_decompress_to_buffer(_bws(cblob, clens)))
    dev = zstd.DeviceBufferWithSegments(torch.from_numpy(cblob).cuda(), _table(clens).tobytes())
    dout = zstd.ZstdDecompressor().multi_decompress_to_buffer(dev)
    assert len(dout) == len(lens)
    assert dout.tobytes() == host
    assert host == blob.tobytes()


# ---------------------------------------------------------------- sub-batches over the pipeline contexts
@pytest.fixture
def small_sub_batches(monkeypatch, auto):
    def set_bytes(n):
        monkeypatch.setattr(zstd.ZstdDecompressor, "SUB_BATCH_INPUT_BYTES", n)
    return set_bytes


def _sub_batches(total_input, n, sub):
    return max(1, min(n // 256 or 1, total_input // sub))


def test_sub_batches_with_a_dictionary_and_exact_sizes(ref, small_sub_batches):
    """4096 records with a trained dictionary in 16 sub-batches over the four contexts, each with its own digest of the
    dictionary; decompressed_sizes sliced per sub-batch."""
    recs = corpus.json_records(4096 + 500)
    dct = ref.train_dictionary(16384, recs[4096:])
    recs = recs[:4096]
    lens = np.array([len(r) for r in recs], dtype=np.uint64)
    blob = np.frombuffer(b"".join(recs), dtype=np.uint8)
    cblob, clens = _compress(ref, blob, lens, level=3, dct=dct)
    small_sub_batches(int(clens.sum()) // 16 + 1)
    assert _sub_batches(int(clens.sum()), len(lens), zstd.ZstdDecompressor.SUB_BATCH_INPUT_BYTES) == 15
    d = zstd.ZstdDecompressor(dict_data=zstd.ZstdCompressionDict(dct))
    out = d.multi_decompress_to_buffer(_bws(cblob, clens), decompressed_sizes=lens.tobytes())
    assert len(out._buffers) == 15
    assert _host_bytes(out) == blob.tobytes()
    _sample(ref, out, cblob, clens, lens, blob, dct=dct, every=301)
    # an exact size that is one byte short is an error of that item, whichever sub-batch holds it
    short = lens.copy(); short[3000] -= 1
    with pytest.raises(zstd.ZstdError, match=r"error decompressing item 3000: "):
        d.multi_decompress_to_buffer(_bws(cblob, clens), decompressed_sizes=short.tobytes())


def _collection(ref, rng, parts):
    """A BufferWithSegmentsCollection of several buffers of 4 KiB-ish text frames; returns it with its pieces."""
    bufs, pieces = [], []
    for n in parts:
        lens = rng.integers(2048, 6000, n).astype(np.uint64)
        blob = _text(int(lens.sum()))
        cblob, clens = _compress(ref, blob, lens, level=3, checksum=True)
        bufs.append(_bws(cblob, clens)); pieces.append((blob, lens, cblob, clens))
    return bufs, pieces


def _damaged(piece, items):
    """The buffer of `piece` with a wrong content checksum on each of `items`."""
    blob, lens, cblob, clens = piece
    bad = cblob.copy()
    for item in items:
        bad[int(_table(clens)[item, 0] + clens[item]) - 2] ^= 0x11
    return _bws(bad, clens)


def test_sub_batches_of_a_collection_raise_the_lowest_global_index(ref, small_sub_batches):
    """Three buffers (1000, 3000 and 2500 frames) cut into sub-batches of 256 KiB of input (3, 11 and 9 of them).  Two
    failing sub-batches of one buffer: the lower item is raised, wherever the pool finishes them.  Failing items in two
    buffers: the first buffer's, with its index in the whole collection."""
    rng = np.random.default_rng(9)
    small_sub_batches(256 << 10)
    bufs, pieces = _collection(ref, rng, (1000, 3000, 2500))
    out = zstd.ZstdDecompressor().multi_decompress_to_buffer(zstd.BufferWithSegmentsCollection(*bufs))
    assert len(out) == 6500 and len(out._buffers) == 3 + 11 + 9
    assert _host_bytes(out) == b"".join(p[0].tobytes() for p in pieces)
    d = zstd.ZstdDecompressor()
    # items 300 and 2700 of the second buffer (global 1300 and 3700): sub-batches of ~270 frames, so about its second and
    # its tenth; whichever is damaged first
    for items in ((300, 2700), (2700, 300)):
        with pytest.raises(zstd.ZstdError, match=r"error decompressing item 1300: Restored data doesn't match checksum"):
            d.multi_decompress_to_buffer(zstd.BufferWithSegmentsCollection(bufs[0], _damaged(pieces[1], items), bufs[2]))
    # item 2700 of the second buffer and item 100 of the third (global 4100)
    with pytest.raises(zstd.ZstdError, match=r"error decompressing item 3700: "):
        d.multi_decompress_to_buffer(zstd.BufferWithSegmentsCollection(bufs[0], _damaged(pieces[1], (2700,)),
                                                                       _damaged(pieces[2], (100,))))
    # only the third buffer's: its own global index
    with pytest.raises(zstd.ZstdError, match=r"error decompressing item 4100: "):
        d.multi_decompress_to_buffer(zstd.BufferWithSegmentsCollection(*bufs[:2], _damaged(pieces[2], (100,))))


def test_second_call_on_the_same_contexts_keeps_the_first_result(ref, small_sub_batches):
    """Two calls of 12 sub-batches each on the same four contexts; the first result is read only after the second call
    returned, and both are intact."""
    rng = np.random.default_rng(12)
    small_sub_batches(192 << 10)
    (b1, b2), pieces = _collection(ref, rng, (3072, 3072))
    d = zstd.ZstdDecompressor()
    out1 = d.multi_decompress_to_buffer(b1)
    out2 = d.multi_decompress_to_buffer(b2)
    assert len(out1._buffers) >= 8 and len(out2._buffers) >= 8
    assert _host_bytes(out1) == pieces[0][0].tobytes()
    assert _host_bytes(out2) == pieces[1][0].tobytes()
    _sample(ref, out1, pieces[0][2], pieces[0][3], pieces[0][1], pieces[0][0], every=257)
