"""The compression kernels' own source, run on the CPU.

tests/host_encoder.build_compress_sim() compiles python_zstandard_b200/csrc/zb_encode.cu (everything above its
launchers: the block kernel with all its phases, the frame layout kernels, XXH64) with g++ on the mini SIMT runtime of
tests/simt.h -- every thread of a CTA is a fiber, __syncthreads and the warp collectives are rendezvous points -- and
drives it the way zb_api.cu does (block jobs, persistent CTAs, slots, frame sizes, scan, frame writer).  The frames go
through the unmodified reference decoder and the oracle.  The device build differs only in timing, so the compressed
bytes are the same except where the link phase lets lanes of one step race for a hash slot (the hardware picks a winner
we cannot predict); sizes are asserted against the reference with the margins the GPU suite uses."""
import ctypes as C
import os

import numpy as np
import pytest

import corpus
from tests import host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")


@pytest.fixture(scope="module")
def sim():
    return host_encoder.build_compress_sim()


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


def compress(sim, segs, checksum=False, content_size=True, n_ctas=2, dual=False, dct=b"", level=None, window_log=0):
    """[frame bytes] for a batch of byte strings through the kernel source.  dual=True: the level >= 4 mode (level 4 unless
    `level` says otherwise); dual=2: the record kernel zb_compress_recs.  window_log 0: the default window."""
    if level is None:
        level = 4 if dual is True or dual == 1 else 3
    blob = b"".join(segs) + bytes(64)
    off = np.cumsum([0] + [len(s) for s in segs[:-1]]).astype(np.uint64)
    ln = np.array([len(s) for s in segs], dtype=np.uint64)
    src = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    cap = sum(len(s) + len(s) // 128 + 64 for s in segs) + 64
    out = (C.c_ubyte * cap)()
    oo = (C.c_uint64 * len(segs))(); ol = (C.c_uint64 * len(segs))()
    dbuf = (C.c_ubyte * (len(dct) + 64)).from_buffer_copy(dct + bytes(64))
    tot = sim.t_compress_batch(C.addressof(src), off.ctypes.data, ln.ctypes.data, len(segs), int(checksum), int(content_size), n_ctas,
                               C.addressof(out), cap, C.addressof(oo), C.addressof(ol), int(dual == 2),
                               C.addressof(dbuf) if dct else None, len(dct), level, window_log)
    assert tot >= 0 and tot == sum(ol)
    assert all(oo[i] == sum(ol[:i]) for i in range(len(segs)))          # frames are packed tightly, in order
    return [bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(len(segs))]


def test_reference_known_answers(sim, ref):
    """Byte-exact frames where the reference's tests pin them (tests/test_compressor_compress.py:19,28,34;
    tests/test_compressor_multi_compress_to_buffer.py:45,64 and the frames SURVEY.md probed)."""
    f = compress(sim, [b"foo" * 12, b"bar" * 6], checksum=True)
    assert f[0] == bytes.fromhex("28b52ffd24244d000018666f6f01008e6e08a788b46f")
    assert len(f[0]) + len(f[1]) == 44 and f[1] == ref.compress(b"bar" * 6, level=3, checksum=True)
    f = compress(sim, [b"foo" * 4, b"bar" * 6], checksum=True)
    assert len(f[0]) + len(f[1]) == 47 and f[0] == ref.compress(b"foo" * 4, level=3, checksum=True)
    assert compress(sim, [b"", b"foo"]) == [bytes.fromhex("28b52ffd2000010000"), bytes.fromhex("28b52ffd2003190000666f6f")]
    assert compress(sim, [b"", b"x"], content_size=False)[0] == bytes.fromhex("28b52ffd0000010000")
    assert len(compress(sim, [b"x" * 64], checksum=True)[0]) <= 21


def test_round_trips_through_the_reference_and_the_oracle(sim, ref):
    from oracle import Oracle
    orc = Oracle()
    rng = np.random.default_rng(41)
    text = corpus.text_corpus(1 << 20)
    segs = [b"a", b"ab" * 5, bytes(9), bytes(text[:300]), bytes(text[1000:1000 + 2047]), bytes(text[5000:5000 + 2048]),
            bytes(text[9000:9000 + 4096]), bytes(40000), rng.integers(0, 256, 20000).astype(np.uint8).tobytes(),
            corpus.binary_blob(30000).tobytes(), bytes(text[20000:20000 + 70000]),
            (b"0123456789abcdef" * 3000) + bytes(text[:777]) + b"0123456789abcdef" * 500]
    for checksum in (False, True):
        frames = compress(sim, segs, checksum=checksum, n_ctas=3)
        for s, f in zip(segs, frames):
            assert ref.decompress(f, len(s)) == s
            assert orc.decompress(f, len(s)) == s
            assert len(f) <= len(s) + len(s) // 128 + 24                 # never much larger than the input
    frames = compress(sim, segs[:6], content_size=False)
    for s, f in zip(segs[:6], frames):
        assert ref.decompress(f, len(s)) == s


def test_multi_block_segments(sim, ref):
    """Segments above 128 KiB are cut into blocks that different CTAs may take; frame headers follow the size class."""
    text = corpus.text_corpus(1 << 20)
    segs = [bytes(text[100000:100000 + 300000]), bytes(text[:131072]), bytes(text[7:7 + 131073])]
    frames = compress(sim, segs, checksum=True, n_ctas=4)
    for s, f in zip(segs, frames):
        assert ref.decompress(f, len(s)) == s
    assert len(frames[1]) <= len(ref.compress(segs[1], level=3, checksum=True)) * 1.06      # single block, GPU-suite margin


def test_sizes_against_the_reference(sim, ref):
    """The size margins of tests/test_gpu_compress.py, on the CPU: 4 KiB text within 2 %, mixed content within 3 %."""
    blob, off, ln = corpus.text_segments(40, 4096)
    segs = [bytes(blob[int(o):int(o) + int(l)]) for o, l in zip(off, ln)]
    ours = sum(len(f) for f in compress(sim, segs, n_ctas=4))
    theirs = sum(len(ref.compress(s, level=3)) for s in segs)
    assert ours <= theirs * 1.02, (ours, theirs)
    mix, off, ln = corpus.silesia_mix(6, 32768)
    segs = [bytes(mix[int(o):int(o) + int(l)]) for o, l in zip(off, ln)]
    frames = compress(sim, segs, n_ctas=3)
    assert all(ref.decompress(f, len(s)) == s for s, f in zip(segs, frames))
    assert sum(map(len, frames)) <= sum(len(ref.compress(s, level=3)) for s in segs) * 1.03


def test_frames_above_two_mebibytes_declare_a_window(sim, ref):
    """Above 2 MiB the header carries a window descriptor (2 MiB, the reference's level-3 window) instead of the
    single-segment flag; the frame still regenerates the input through the reference decoder."""
    data = bytes(3 << 20)
    f = compress(sim, [data], checksum=True, n_ctas=4)[0]
    theirs = ref.compress(data, level=3, checksum=True)
    assert f[:10] == theirs[:10] and (f[4] >> 5) & 1 == 0 and f[5] == (21 - 10) << 3
    assert ref.decompress(f, len(data)) == data


def test_dual_table_mode(sim, ref):
    """Level >= 4 runs the two-table match finder (4-byte and 8-byte hash heads in the same shared memory): valid frames,
    never larger than the single-table parse by more than noise, and at the reference's level-3 size or below on text
    (CPU model tools/enc_model3.c predicted it)."""
    text = corpus.text_corpus(1 << 20)
    rng = np.random.default_rng(43)
    segs = [bytes(text[:131072]), bytes(text[500000:500000 + 4096]), bytes(text[600000:600000 + 4096]), bytes(text[1234:1234 + 1500]),
            b"foo" * 12, b"", bytes(9000), rng.integers(0, 256, 5000).astype(np.uint8).tobytes(), bytes(text[700000:700000 + 200000])]
    one = compress(sim, segs, checksum=True, n_ctas=3, dual=False)
    two = compress(sim, segs, checksum=True, n_ctas=3, dual=True)
    for s, f in zip(segs, two):
        assert ref.decompress(f, len(s)) == s if s else len(f) == 13
    assert sum(map(len, two)) < sum(map(len, one))
    theirs = [len(ref.compress(segs[i], level=3, checksum=True)) for i in (0, 1, 2)]
    assert sum(len(two[i]) for i in (0, 1, 2)) <= sum(theirs) * 1.005
    assert all(len(two[i]) <= t * 1.04 for i, t in zip((0, 1, 2), theirs))           # single 4 KiB segments scatter by a few %
    assert len(two[0]) <= len(one[0]) * 0.98                      # 128 KiB text: at least 2 % smaller than the single table


def test_dictionary_compression(sim, ref):
    """Config 4 on the CPU build: records against a trained dictionary (digest, hash table and CTables built by the
    library's own kernels).  Frames carry the dictionary id, regenerate through the reference decoder and the oracle with
    the dictionary, reuse its entropy tables (repeat modes / treeless literals) and land within 3 % of the reference's
    size with the same dictionary; a long input whose first match reaches back into the dictionary works too."""
    from oracle import Oracle
    orc = Oracle()
    recs = corpus.json_records(470)
    dct = ref.train_dictionary(16384, recs[:400])
    sample = recs[400:] + [recs[5] * 40]
    frames = compress(sim, sample, checksum=True, n_ctas=3, dct=dct)
    ours = theirs = plain = 0
    for r, f in zip(sample, frames):
        assert ref.decompress(f, len(r), dct) == r and orc.decompress(f, len(r), dct) == r
        assert f[4] & 3 != 0                                       # dictionary id present
        ours += len(f); theirs += len(ref.compress(r, level=3, dict_data=dct, checksum=True))
    plain = sum(map(len, compress(sim, sample, checksum=True, n_ctas=3)))
    assert ours < plain * 0.8 and ours <= theirs * 1.03, (ours, theirs, plain)


def test_two_table_mode_uses_the_previous_block_as_history(sim, ref):
    """In the level >= 4 mode a block that is not the first of its frame links into the last 32 KiB of the block in front
    of it: multi-block frames stay valid (reference decoder, oracle) and shrink from +7.6 % to about +1 % of the
    reference's level 3 on 300 KB of text."""
    from oracle import Oracle
    orc = Oracle()
    text = corpus.text_corpus(4 << 20)
    segs = [bytes(text[100000:100000 + 300000]), bytes(text[1000000:1000000 + 131073]), bytes(270000)]
    one = compress(sim, segs, checksum=True, n_ctas=3, dual=False)
    two = compress(sim, segs, checksum=True, n_ctas=3, dual=True)
    for s, f in zip(segs, two):
        assert ref.decompress(f, len(s)) == s and orc.decompress(f, len(s)) == s
    theirs = len(ref.compress(segs[0], level=3, checksum=True))
    assert len(two[0]) <= theirs * 1.02 and len(two[0]) <= len(one[0]) * 0.96


# ---------------------------------------------------------------------------------------------------------------------
# The round-2 kernel (zb_compress_smem: one CTA of 1024 threads per block, the block resident in shared memory, serial hash
# links beside warp-per-region verify + parse, sub-blocks with their FSE state chains side by side).  The launcher gives
# it every call whose largest block is >= 8 KiB (no dictionary, level-3 class).
def compress_smem(sim, segs, checksum=False, n_ctas=2, content_size=True, level=3, window_log=0):
    blob = b"".join(segs) + bytes(64)
    off = np.cumsum([0] + [len(s) for s in segs[:-1]]).astype(np.uint64)
    ln = np.array([len(s) for s in segs], dtype=np.uint64)
    src = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    cap = sum(len(s) + len(s) // 128 + 64 for s in segs) + 64
    out = (C.c_ubyte * cap)()
    oo = (C.c_uint64 * len(segs))(); ol = (C.c_uint64 * len(segs))()
    tot = sim.t_compress_batch2(C.addressof(src), off.ctypes.data, ln.ctypes.data, len(segs), int(checksum), int(content_size), n_ctas,
                                C.addressof(out), cap, C.addressof(oo), C.addressof(ol), level, window_log)
    assert tot >= 0 and tot == sum(ol)
    return [bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(len(segs))]


def test_smem_kernel_round_trips_and_sizes(sim, ref):
    """Frames of the shared-memory kernel regenerate through the reference decoder and the oracle; sizes stay inside the
    margins stated in DESIGN.md (128 KiB text <= +2.5 %, mix <= +1.5 %, multi-block inputs <= +5 % -- blocks are independent)."""
    from oracle import Oracle
    orc = Oracle()
    rng = np.random.default_rng(7)
    text = corpus.text_corpus(2 << 20).tobytes()
    b, o, l = corpus.silesia_mix(10, 131072)
    mix = [bytes(b[int(a):int(a) + int(c)]) for a, c in zip(o, l)]
    odd = [text[7:7 + 131071], text[300001:300001 + 9000], bytes(131072), b"ab" * 40000, rng.integers(0, 256, 70000).astype(np.uint8).tobytes(),
           (b"0123456789abcdef" * 3000) + text[:777] + b"0123456789abcdef" * 500, text[5:5 + 300000], text[11:11 + 131073]]
    for segs, margin in ((mix, 1.015), ([text[i * 131072:(i + 1) * 131072] for i in range(4)], 1.025), (odd, None)):
        for checksum in ((False, True) if margin is None else (False,)):
            frames = compress_smem(sim, segs, checksum=checksum, n_ctas=3)
            for s, f in zip(segs, frames):
                assert ref.decompress(f, len(s)) == s
                assert orc.decompress(f, len(s)) == s
                assert len(f) <= len(s) + len(s) // 128 + 24 + 3 * (len(s) >> 17)
        if margin is not None:
            ours = sum(map(len, frames)); theirs = sum(len(ref.compress(s, level=3)) for s in segs)
            assert ours <= theirs * margin, (ours, theirs)


def test_record_kernel_with_dictionary(sim, ref):
    """zb_compress_recs (a warp per record, dictionary staged in shared memory: BASELINE config 4): frames regenerate through
    the reference decoder with the dictionary, sizes stay within +1 % of the reference's level 3 with the same dictionary
    on JSON-like records; records the dictionary does not help, empty, tiny, run and random records ride along."""
    recs = corpus.json_records(2400)
    dct = ref.train_dictionary(112640, recs[:2000])
    recs = recs[2000:]
    frames = compress(sim, recs, n_ctas=2, dual=2, dct=dct)
    for s, f in zip(recs, frames):
        assert ref.decompress(f, len(s), dict_data=dct) == s
    ours = sum(map(len, frames)); theirs = sum(len(ref.compress(s, level=3, dict_data=dct)) for s in recs)
    assert ours <= theirs * 1.01, (ours, theirs)
    text = corpus.text_corpus(1 << 20).tobytes()
    odd = [b"", b"a", b"abc" * 100, bytes(2048), np.random.default_rng(1).integers(0, 256, 2048).astype(np.uint8).tobytes(),
           text[:2048], text[5000:5000 + 1399], recs[3] + recs[4][:2048 - len(recs[3])], dct[-700:], dct[-2048:]]
    for checksum in (False, True):
        frames = compress(sim, odd, n_ctas=1, dual=2, dct=dct, checksum=checksum)
        for s, f in zip(odd, frames):
            assert ref.decompress(f, len(s), dict_data=dct) == s
            assert len(f) <= len(s) + 24
