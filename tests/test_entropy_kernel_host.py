"""The decode kernels' own source, run on the CPU.

tests/host_encoder.build_sim() compiles python_zstandard_b200/csrc/zb_decode.cu and zb_entropy.cuh whole on the SIMT
runtime of tests/simt.h.  t_decode_frame runs a frame through the launchers as the library runs a batch of one: dictionary
digest, frame scan, placement, and the whole lane-per-frame entropy kernel (block loop, literal sections, sequence headers,
table builds, the 3-state sequence stream, repcode history, every validity check) on one CTA of 7 warps, with the warp
collectives of the device.  A serial loop replays the block / sequence / literal records the way the execute kernels read
them, and the bytes must equal the reference's.  With one frame per call the other 31 lanes of its warp are idle: the
interplay of busy lanes (pool claims, second passes) and the execute kernels themselves are covered by the batch tests
(test_decode_pipeline_host.py, test_crafted_frames_host.py) and the GPU suite."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import helpers, host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")
PAD = 64


@pytest.fixture(scope="module")
def kern():
    return host_encoder.build_sim()


def decode(kern, frame, cap, dct=b""):
    """(status, bytes, n_blocks, n_seq) of one frame through the kernel source."""
    src = (C.c_ubyte * (len(frame) + 2 * PAD))()                 # the bit reader loads aligned words around a stream
    C.memmove(C.addressof(src) + PAD, frame, len(frame))
    dbuf = (C.c_ubyte * (len(dct) + 2 * PAD))()
    if dct:
        C.memmove(C.addressof(dbuf) + PAD, dct, len(dct))
    out = (C.c_ubyte * (cap + 2 * PAD))()
    out_n, nb, ns = C.c_uint64(0), C.c_uint32(0), C.c_uint32(0)
    rc = kern.t_decode_frame(C.addressof(src) + PAD, len(frame), (C.addressof(dbuf) + PAD) if dct else None, len(dct),
                             C.addressof(out) + PAD, cap, C.byref(out_n), C.byref(nb), C.byref(ns))
    assert bytes(out[:PAD]) == bytes(PAD) and bytes(out[PAD + cap:]) == bytes(PAD)      # nothing written outside dst
    return rc, bytes(out[PAD:PAD + out_n.value]), nb.value, ns.value


def test_known_answer_frames(kern):
    assert decode(kern, helpers.KAT_EMPTY_NOFCS, 16)[:2] == (0, b"")
    assert decode(kern, helpers.KAT_EMPTY_FCS, 16)[:2] == (0, b"")
    assert decode(kern, helpers.KAT_FOO, 16)[:2] == (0, b"foo")
    rc, got, nb, ns = decode(kern, helpers.KAT_LARGE, 131073)
    assert (rc, got, nb, ns) == (0, b"f" * 131072 + b"o", 2, 1)


def test_golden_vectors(kern):
    """Every committed reference-made frame (levels -5..19, checksums, multi-block, no content size, RLE and raw blocks,
    trained dictionary) regenerates bit-exact."""
    vecs = helpers.golden_vectors()
    assert len(vecs) >= 16
    for name, frame, raw, dct in vecs:
        rc, got, nb, ns = decode(kern, frame, len(raw), dct)
        assert rc == 0 and got == raw, name


def test_live_reference_frames(kern):
    """Frames made now by the unmodified reference: text, JSON records, binary, at several levels and sizes, with and
    without a dictionary; block types and sequence-table modes of all kinds occur."""
    import corpus
    from oracle import RefZstd
    ref = RefZstd()
    blob = corpus.text_corpus(1 << 20)
    recs = corpus.json_records(600)
    dct = ref.train_dictionary(16384, recs[:400])
    rng = np.random.default_rng(31)
    cases = []
    for size in (1, 17, 300, 4096, 70000, 300000):
        o = int(rng.integers(0, len(blob) - size))
        cases.append(bytes(blob[o:o + size]))
    cases.append(corpus.binary_blob(50000).tobytes())
    cases.append(bytes(40000))
    cases.append(rng.integers(0, 256, 30000).astype(np.uint8).tobytes())
    cases.append((b"abcdefgh" * 5000) + bytes(rng.integers(0, 256, 100).astype(np.uint8)) + b"abcdefgh" * 3000)
    seqs_seen = blocks_seen = 0
    for data in cases:
        for level in (-3, 1, 3, 7, 19):
            frame = ref.compress(data, level=level, checksum=bool(level & 1))
            rc, got, nb, ns = decode(kern, frame, len(data))
            assert rc == 0 and got == data, (len(data), level)
            seqs_seen += ns; blocks_seen += nb
    for r in recs[400:440]:
        frame = ref.compress(r, level=3, dict_data=dct)
        rc, got, _, _ = decode(kern, frame, len(r), dct)
        assert rc == 0 and got == r
        rc, got, _, _ = decode(kern, frame, len(r))              # without the dictionary the frame cannot regenerate r
        assert rc != 0 or got != r
    assert seqs_seen > 20000 and blocks_seen > 60


def test_corrupt_frames_follow_the_reference(kern):
    """Single-bit corruptions of frames without a content checksum (so that the reference accepts many of them):
    whatever the reference rejects the kernel code rejects; when both accept, the bytes are the same; the kernel code may
    reject more (it demands that every literal stream is consumed exactly, the reference's fast loop does not)."""
    import corpus
    from oracle import RefZstd
    ref = RefZstd()
    blob = corpus.text_corpus(1 << 20)
    rng = np.random.default_rng(32)
    both = ref_rejects = stricter = 0
    for size, level in ((600, 3), (5000, 3), (5000, 1), (40000, 5), (140000, 3)):
        o = int(rng.integers(0, len(blob) - size))
        data = bytes(blob[o:o + size])
        frame = ref.compress(data, level=level, checksum=False)
        for _ in range(200):
            bad = bytearray(frame)
            k = int(rng.integers(4, len(bad)))
            bad[k] ^= 1 << int(rng.integers(0, 8))
            try:
                want = ref.decompress(bytes(bad), len(data))
            except RefZstd.Error:
                want = None
            rc, got, _, _ = decode(kern, bytes(bad), len(data))
            if want is None:
                assert rc != 0, (size, level, k)
                ref_rejects += 1
            elif rc == 0:
                assert got == want, (size, level, k)
                both += 1
            else:
                stricter += 1
    assert ref_rejects > 200 and both > 100 and stricter < both
