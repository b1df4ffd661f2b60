"""The output chunks of a batch decode, on the CPU.

run_decompress (zb_api.cu) cuts a call whose output is copied back to the host into chunks of frames: the copy of chunk k
overlaps the kernels of chunk k + 1.  The cuts are by frame count; every chunk has its own work counter, its own entropy
launch shape (warps per CTA, frames per warp, CTAs) from its own average output size, its own execute range -- frames,
blocks or output bytes -- and its own checksum pass (zb_chunk_count, zb_chunk_cut, zb_chunk_shape in zb_common.cuh).

tests/host_encoder.build_decode_sim() runs the same plan chunk by chunk on the CPU build of the kernels (`chunk_bytes`
stands for ZB200_OUT_CHUNK_BYTES).  It copies each chunk's output range out as soon as the chunk's kernels are done, and
assembles the result from those copies alone; then it overwrites the range in its working buffer, so any later write
there -- even of the right bytes -- is counted.  Every test runs on the three execute paths, and checks the bytes against
the source, the reference and the oracle, the status of every frame, and the plan itself."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

import corpus
from tests import host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")
PAD = 64
SMS = 1          # the SM count the plan shapes the entropy launches for: 1 CTA of 7 or 8 warps keeps `take` above 1


@pytest.fixture(scope="module", params=["lane-per-frame", "lane-per-block", "lane-per-block+pointer-jumping"])
def sim(request):
    L = host_encoder.build_decode_sim()
    L.t_set_block_path({"lane-per-frame": 0, "lane-per-block": 1}.get(request.param, 2))
    L.path = request.param
    yield L
    L.t_set_block_path(0)


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


@pytest.fixture(scope="module")
def orc():
    from oracle import Oracle
    return Oracle()


class Run:
    def __init__(self, outs, st, plan):
        self.outs, self.st = outs, st
        self.n_chunks, self.changed, self.redone = int(plan[0]), int(plan[1]), int(plan[2])
        c = [plan[3 + 5 * k:8 + 5 * k] for k in range(self.n_chunks)]
        self.cut = [int(x[0]) for x in c] + [len(st)]
        self.shape = [(int(x[1]), int(x[2]), int(x[3])) for x in c]         # (warps, take, ctas); 0s on the block path
        self.out_bytes = [int(x[4]) for x in c]


def decompress(sim, frames, sizes, chunk_bytes, dct=b"", exact_sizes=False):
    blob = bytes(PAD) + b"".join(frames) + bytes(PAD)
    off = (np.cumsum([0] + [len(f) for f in frames[:-1]]) + PAD).astype(np.uint64)
    ln = np.array([len(f) for f in frames], dtype=np.uint64)
    src = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    dbuf = (C.c_ubyte * (len(dct) + 2 * PAD)).from_buffer_copy(bytes(PAD) + dct + bytes(PAD))
    cap = sum(sizes) + 64
    out = (C.c_ubyte * cap)()
    n = len(frames)
    oo = (C.c_uint64 * n)(); ol = (C.c_uint64 * n)(); st = (C.c_uint32 * n)()
    want = (C.c_uint64 * n)(*sizes)
    plan = (C.c_uint64 * (3 + 5 * 33))()
    tot = sim.t_decompress_batch(C.addressof(src), off.ctypes.data, ln.ctypes.data, n, (C.addressof(dbuf) + PAD) if dct else None, len(dct),
                                 SMS, 8, 32, C.addressof(out), cap, C.addressof(oo), C.addressof(ol), C.addressof(st),
                                 C.addressof(want) if exact_sizes else None, chunk_bytes, C.addressof(plan))
    assert tot >= 0
    r = Run([bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(n)], list(st), plan)
    # what holds for every call: the copies were all the caller got, and nothing touched a chunk after its copy
    assert r.changed == 0, "later chunks wrote %d bytes of earlier chunks" % r.changed
    assert r.redone == 0, "later chunks decoded %d frames of earlier chunks again" % r.redone
    assert r.cut == [n * k // r.n_chunks for k in range(r.n_chunks)] + [n]
    return r


def _with_tail(body, period=b"0123456789abcdef"):
    """Content that ends in a repeated pattern, so the frame ends with a match: its last output byte has a source
    (the pointer-jumping stage's gather writes it) and the chunk border falls behind a match."""
    return body + period * 40


def _mixed(ref, text, rng):
    """Six groups of 8 frames, each group one chunk when the batch is cut in six; adjacent groups differ in average
    size, so their entropy launches differ in shape.  Small frames (1 B .. 4 KiB: the tile executor), 100 KiB, 6 KiB,
    24 KiB, small again, then frames of several blocks (two of ~1 MiB)."""
    def piece(size):
        o = int(rng.integers(0, len(text) - size - 1))
        return _with_tail(bytes(text[o:o + max(size - 640, 0)]))[:size] if size > 700 else bytes(text[o:o + size])
    groups = [[1, 37, 700, 2000, 4096, 3000, 1500, 4000],
              [100 << 10] * 8,
              [6 << 10] * 8,
              [24 << 10] * 8,
              [9, 4096, 333, 2500, 1024, 4095, 64, 3900],
              [1 << 20, 150 << 10, 200 << 10, 1000 << 10, 140 << 10, 160 << 10, 131 << 10, 135 << 10]]
    segs = [piece(s) for g in groups for s in g]
    frames = [ref.compress(s, level=1 + i % 5, checksum=i % 3 == 0) for i, s in enumerate(segs)]
    return segs, frames


@pytest.fixture(scope="module")
def mixed(ref):
    return _mixed(ref, corpus.text_corpus(4 << 20), np.random.default_rng(2024))


def _check(ref, orc, r, segs, frames, bad=(), dct=b""):
    for i, s in enumerate(segs):
        if i in bad:
            assert r.st[i] != 0, i
            continue
        assert r.st[i] == 0 and r.outs[i] == s, i
    for i in range(0, len(segs), 7):                # the reference and the oracle on a sample
        if i not in bad:
            assert r.outs[i] == ref.decompress(frames[i], len(segs[i]), dct) == orc.decompress(frames[i], len(segs[i]), dct), i


def _assert_shapes(sim, r, want):
    """The chunks' lane-per-frame entropy launches; the block path has one launch for all blocks instead."""
    if sim.path == "lane-per-frame":
        assert r.shape == want
    else:
        assert r.shape == [(0, 0, 0)] * r.n_chunks


def test_chunk_per_size_group(sim, ref, orc, mixed):
    """Six chunks of eight frames: warps per CTA alternate 8 (small frames) and 7.  Eight frames are spread over the
    warps of one SM: 8 warps take 1 frame each, 7 warps 2 (below the 8, 3 and 3 that the sizes alone would give)."""
    segs, frames = mixed
    total = sum(map(len, segs))
    r = decompress(sim, frames, [len(s) for s in segs], total // 6)
    assert r.n_chunks == 6 and r.cut == [0, 8, 16, 24, 32, 40, 48]
    assert r.out_bytes == [sum(map(len, segs[8 * k:8 * k + 8])) for k in range(6)]
    _assert_shapes(sim, r, [(8, 1, 1), (7, 2, 1), (8, 1, 1), (7, 2, 1), (8, 1, 1), (7, 2, 1)])
    _check(ref, orc, r, segs, frames)


def test_take_follows_each_chunks_own_average(sim, ref, orc):
    """Four chunks of 64 frames: up to 4 KiB, 20 KiB, 12 KiB and 40 KiB.  With that many frames per chunk the sizes, not
    the spread over the warps, set `take` where they ask for fewer than 64 / 7: 8 frames per warp for 20 KiB frames, 4 for
    40 KiB ones.  The 12 KiB chunk would take 16 and is spread to 10, the small one would take 32 and is spread to 8.  The
    batch's average (~18 KiB) would give 8 to every chunk."""
    text = corpus.text_corpus(4 << 20)
    rng = np.random.default_rng(64)
    sizes = [int(x) for x in rng.integers(1, 4097, 64)] + [20 << 10] * 64 + [12 << 10] * 64 + [40 << 10] * 64
    segs = []
    for size in sizes:
        o = int(rng.integers(0, len(text) - size - 1))
        segs.append(_with_tail(bytes(text[o:o + size - 640]))[:size] if size > 700 else bytes(text[o:o + size]))
    frames = [ref.compress(s, level=1 + i % 5, checksum=i % 4 == 0) for i, s in enumerate(segs)]
    r = decompress(sim, frames, sizes, sum(sizes) // 4)
    assert r.n_chunks == 4 and r.cut == [0, 64, 128, 192, 256]
    _assert_shapes(sim, r, [(8, 8, 1), (7, 8, 1), (7, 10, 1), (7, 4, 1)])
    _check(ref, orc, r, segs, frames)


def test_every_frame_its_own_chunk(sim, ref, orc, mixed):
    """More chunks asked for than there are frames: the count is clamped to the frame count, one frame per chunk."""
    segs, frames = mixed
    segs, frames = segs[:4] + segs[8:11] + segs[16:19] + segs[40:42], frames[:4] + frames[8:11] + frames[16:19] + frames[40:42]
    r = decompress(sim, frames, [len(s) for s in segs], 1)
    assert r.n_chunks == len(segs) == 12 and r.cut == list(range(13))
    assert r.out_bytes == [len(s) for s in segs]
    _check(ref, orc, r, segs, frames)


def _empty(ref, k):
    """Frames that regenerate nothing: an empty frame, or a skippable frame in front of one."""
    e = ref.compress(b"", level=3, checksum=k % 2 == 1)
    return e if k % 3 else struct.pack("<II", 0x184D2A50, 5 + k) + bytes(range(5 + k)) + e


def test_thirty_two_chunks_with_empty_ones(sim, ref, orc):
    """48 frames cut in the 32 chunks of the cap (one or two frames each, cut[k] = 48k / 32); the chunks [1, 3), [10, 12)
    and the last, [46, 48), hold only frames without output, so their output range is empty."""
    text = corpus.text_corpus(1 << 20)
    rng = np.random.default_rng(7)
    empty = {1, 2, 10, 11, 46, 47}
    segs, frames = [], []
    for i in range(48):
        if i in empty:
            segs.append(b""); frames.append(_empty(ref, i))
            continue
        size = int(rng.choice([300, 4000, 9000, 30000, 140000]))
        o = int(rng.integers(0, len(text) - size))
        segs.append(_with_tail(bytes(text[o:o + size])))
        frames.append(ref.compress(segs[-1], level=int(rng.integers(1, 6)), checksum=bool(i % 2)))
    r = decompress(sim, frames, [len(s) for s in segs], 1)
    assert r.n_chunks == 32
    assert r.cut[:4] == [0, 1, 3, 4] and r.cut[-2:] == [46, 48]
    assert r.out_bytes[1] == r.out_bytes[7] == r.out_bytes[31] == 0 and r.cut[7] == 10
    _check(ref, orc, r, segs, frames)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_damaged_frames_in_a_chunk(sim, ref, orc, mixed, where):
    """A corrupt frame, a truncated one and one with a wrong checksum, all in the first, a middle or the last of six
    chunks: each keeps its own status, the lowest index is the one reported, every other frame's bytes are exact."""
    segs, frames = mixed
    frames = list(frames)
    base = {"first": 0, "middle": 24, "last": 40}[where]
    wrong, corrupt = [i for i in range(base, base + 8) if i % 3 == 0][:2]      # checksummed: any damage is caught
    cut_short = base + 7
    f = bytearray(frames[corrupt]); f[len(f) // 2] ^= 0x24; frames[corrupt] = bytes(f)
    frames[cut_short] = frames[cut_short][:len(frames[cut_short]) * 2 // 3]
    f = bytearray(frames[wrong]); f[-1] ^= 0x80; frames[wrong] = bytes(f)
    total = sum(map(len, segs))
    r = decompress(sim, frames, [len(s) for s in segs], total // 6)
    assert r.n_chunks == 6
    _check(ref, orc, r, segs, frames, bad={corrupt, cut_short, wrong})
    assert r.st[wrong] == 22                                               # checksum_wrong, from the chunk's own verify pass
    assert min(i for i, s in enumerate(r.st) if s) == wrong


def test_dictionary_checksums_and_exact_sizes(sim, ref, orc):
    """A trained dictionary, checksummed frames and decompressed_sizes given with exact sizes, over 9 chunks of records
    and 40 KiB documents."""
    recs = corpus.json_records(560)
    dct = ref.train_dictionary(16384, recs[:400])
    text = corpus.text_corpus(1 << 20)
    docs = [bytes(text[i * 41000:i * 41000 + 40000 + 17 * i]) for i in range(18)]
    segs = recs[400:490] + docs[:9] + recs[490:560] + docs[9:]
    frames = [ref.compress(s, level=3, dict_data=dct, checksum=i % 2 == 0) for i, s in enumerate(segs)]
    r = decompress(sim, frames, [len(s) for s in segs], sum(map(len, segs)) // 9, dct=dct, exact_sizes=True)
    assert r.n_chunks == 9
    _check(ref, orc, r, segs, frames, dct=dct)
