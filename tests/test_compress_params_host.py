"""The compression kernels across levels, window logs and dictionaries, on the CPU build (tests/host_encoder.py).

The jobs are cut as the launcher cuts them (zb_cut_blocks: blocks of min(2^window_log, 128 KiB)) and the frames are laid
out with the call's level and window_log, so this reaches what a ZstdCompressionParameters(compression_level=L,
window_log=W) call runs on the device.  Every frame must regenerate through the reference decoder, stay within
ZSTD_compressBound and pass tests/frame_check.py -- which also holds every match to the window the header declares, a rule
the in-memory decoders never check.

The batches are built to catch history that leaks across a frame's border: the first segment sits at offset 0 of the
input, with a copy of its own bytes in the memory in front of it, and another segment repeats its predecessor exactly, so
a block that looks in front of its frame finds matches there."""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

import corpus
from tests import host_encoder
from tests.frame_check import check_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")

TEXT = corpus.text_corpus(1 << 20).tobytes()
GUARD = 1 << 16                 # bytes of input memory in front of the first segment


@pytest.fixture(scope="module")
def sim():
    return host_encoder.build_sim()


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


@pytest.fixture(scope="module")
def orc():
    from oracle import Oracle
    return Oracle()


def run(sim, segs, level, window_log, checksum, content_size, dct=b"", smem=False, n_ctas=3):
    """[frame] of a batch through t_compress_batch (t_compress_batch2 when smem).  The first segment starts at offset 0
    of the input pointer; the GUARD bytes in front of it repeat its beginning."""
    body = b"".join(segs)
    front = (segs[0] * (GUARD // max(len(segs[0]), 1) + 1))[:GUARD] if segs[0] else bytes(GUARD)
    blob = front + body + bytes(64)
    buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    src = C.addressof(buf) + GUARD
    off = np.cumsum([0] + [len(s) for s in segs[:-1]]).astype(np.uint64)
    ln = np.array([len(s) for s in segs], dtype=np.uint64)
    cap = sum(len(s) + len(s) // 128 + 64 for s in segs) + 64
    out = (C.c_ubyte * cap)()
    oo = (C.c_uint64 * len(segs))(); ol = (C.c_uint64 * len(segs))()
    if smem:
        tot = sim.t_compress_batch2(src, off.ctypes.data, ln.ctypes.data, len(segs), int(checksum), int(content_size), n_ctas,
                                    C.addressof(out), cap, C.addressof(oo), C.addressof(ol), level, window_log)
    else:
        dbuf = (C.c_ubyte * (len(dct) + 64)).from_buffer_copy(dct + bytes(64))
        tot = sim.t_compress_batch(src, off.ctypes.data, ln.ctypes.data, len(segs), int(checksum), int(content_size), n_ctas,
                                   C.addressof(out), cap, C.addressof(oo), C.addressof(ol), 0,
                                   C.addressof(dbuf) if dct else None, len(dct), level, window_log)
    assert tot >= 0 and tot == sum(ol)
    return [bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(len(segs))]


def block_of(window_log):
    return 1 << window_log if window_log and window_log < 17 else 128 << 10


def batch(window_log, full=True):
    """Segments around the block size B: text of 2B bytes first (two blocks, at offset 0), the same bytes again, text of
    3B + 5, B - 1, B and B + 1 bytes, zeros (RLE blocks), random bytes (raw blocks) and an empty one.  full=False: the
    B + 1 text and its repeat only (header variants)."""
    B = block_of(window_log)
    rng = np.random.default_rng(window_log)
    if not full:
        s = TEXT[7:7 + B + 1]
        return [s, s]
    two = TEXT[1000:1000 + 2 * B]
    return [two, two, TEXT[500000:500000 + 3 * B + 5], TEXT[200000:200000 + B - 1], TEXT[300000:300000 + B],
            TEXT[400000:400000 + B + 1], bytes(B + 1), rng.integers(0, 256, B + 1).astype(np.uint8).tobytes(), b""]


def check(ref, orc, segs, frames, checksum, content_size, dct=b"", dict_id=0):
    found = []
    for i, (s, f) in enumerate(zip(segs, frames)):
        assert ref.decompress(f, len(s), dct) == s, "segment %d" % i
        assert len(f) <= ref.Z.ZSTD_compressBound(len(s)), (i, len(f), len(s))
        found.append(check_frame(f, s, dct, checksum=checksum, content_size=content_size, dict_id=dict_id, oracle=orc))
    return found


# Frames of the parent commit for the windows whose two-table history already stayed inside the frame and the window:
# sha256 over the frames of batch(W) with checksum and content size on, level 4.
PINNED = {
    0: "11b9b1e70bdb470acf3bdde6bd882506baf9f24b679735f930019a64c2a1028b",
    16: "d4d571ebe134b93f01df5c7865a952de8cf06c2efc2365d41f6cdf0a7b5a95f1",
    17: "59dd246a7222555552ca5207d3c634bf2819e2511a882294ad94a034f5755b91",
    18: "d09170c8f505d0b712dfb135ce26b321ede15edb7526cb7fe9505cb676889931",
}

WINDOW_LOGS = [0, 10, 11, 12, 13, 14, 15, 16, 17, 18]


@pytest.mark.parametrize("dual", [False, True], ids=["level3", "level4"])
@pytest.mark.parametrize("window_log", WINDOW_LOGS)
def test_levels_and_window_logs(sim, ref, orc, dual, window_log):
    """Both parse modes at every window log the launcher cuts differently, with and without content size and checksum:
    blocks of at most min(2^W, 128 KiB), a window descriptor (or single segment) that covers every match, and no match
    that reaches in front of its frame."""
    level = 4 if dual else 3
    B = block_of(window_log)
    for checksum, content_size in ((True, True), (False, True), (True, False), (False, False)):
        segs = batch(window_log, full=(checksum, content_size) == (True, True))
        frames = run(sim, segs, level, window_log, checksum, content_size)
        found = check(ref, orc, segs, frames, checksum, content_size)
        for s, h in zip(segs, found):
            assert all(b <= B for b in h["blocks"]) and len(h["blocks"]) == max(1, -(-len(s) // B))
            if content_size and window_log:
                assert h["single"] == (len(s) <= 1 << window_log)
        if dual and window_log in PINNED and (checksum, content_size) == (True, True):
            assert hashlib.sha256(b"".join(frames)).hexdigest() == PINNED[window_log]


@pytest.mark.parametrize("window_log", [13, 14, 15, 16])
def test_smem_kernel_window_logs(sim, ref, orc, window_log):
    """zb_compress_smem, which the launcher gives level-3 calls whose largest block is 8 KiB or more: 8 to 64 KiB blocks."""
    for checksum, content_size in ((True, True), (False, False)):
        segs = batch(window_log, full=checksum)
        frames = run(sim, segs, 3, window_log, checksum, content_size, smem=True)
        found = check(ref, orc, segs, frames, checksum, content_size)
        assert all(b <= 1 << window_log for h in found for b in h["blocks"])


def _raw_dict():
    return TEXT[600000:600000 + 20000]


def _trained_dict():
    return open(os.path.join(ROOT, "tests", "golden", "dict.bin"), "rb").read()


@pytest.mark.parametrize("kind", ["raw", "trained"])
@pytest.mark.parametrize("window_log", [0, 10, 13, 15, 16])
def test_dictionaries_in_the_two_table_mode(sim, ref, orc, kind, window_log):
    """Level 4 with a dictionary: the first block of a frame may reach into the dictionary content (beyond the window --
    RFC 8878 lets a frame reference its dictionary whatever the window), later blocks only into their own frame."""
    import struct
    dct = _raw_dict() if kind == "raw" else _trained_dict()
    dict_id = struct.unpack_from("<I", dct, 4)[0] if kind == "trained" else 0
    B = block_of(window_log)
    recs = corpus.json_records(40)
    segs = [b"".join(recs[:30])[:3 * B + 5], recs[30], recs[31] * 3, dct[-3000:] + TEXT[:2 * B], dct[-3000:] + TEXT[:2 * B]]
    for checksum, content_size in ((True, True), (False, False)):
        frames = run(sim, segs, 4, window_log, checksum, content_size, dct=dct)
        found = check(ref, orc, segs, frames, checksum, content_size, dct, dict_id)
        assert found[3]["max_offset"] > 0
