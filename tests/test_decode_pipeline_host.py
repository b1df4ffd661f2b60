"""All decompression kernels, run on the CPU kernel by kernel the way zb_api.cu launches them.

tests/host_encoder.build_sim() compiles zb_decode.cu + zb_entropy.cuh (frame scan, placement scans, the
lane-per-frame entropy kernel with its shared-memory pool claims, both execute kernels with their dependency frontier,
checksum verification, finish, and their launchers) on the mini SIMT runtime of tests/simt.h: 32 lanes per warp in lock step at every
collective, 7 or 8 warps per CTA, persistent CTAs pulling frames from the work counter.  Output must equal the
reference's, per-frame status codes must match what the GPU suite expects."""
import ctypes as C
import os

import numpy as np
import pytest

import corpus
from tests import helpers, host_encoder

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")
PAD = 64


@pytest.fixture(scope="module", params=["lane-per-frame", "lane-per-block", "lane-per-block+pointer-jumping"])
def sim(request):
    """Every test runs twice: through zb_entropy_decode (a lane per frame) and through the block-parallel path
    (zb_scan_blocks -> zb_entropy_blocks -> zb_resolve_blocks -> zb_patch_blocks: a lane per block, symbolic repcodes)."""
    L = host_encoder.build_sim()
    L.t_set_block_path({"lane-per-frame": 0, "lane-per-block": 1}.get(request.param, 2))
    yield L
    L.t_set_block_path(0)


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


def decompress(sim, frames, sizes, dct=b"", n_ctas=1, warps=8, take=32, exact_sizes=False):
    """(outputs, statuses) of a batch of frames through the kernels, in one chunk."""
    blob = bytes(PAD) + b"".join(frames) + bytes(PAD)
    off = (np.cumsum([0] + [len(f) for f in frames[:-1]]) + PAD).astype(np.uint64)
    ln = np.array([len(f) for f in frames], dtype=np.uint64)
    src = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    dbuf = (C.c_ubyte * (len(dct) + 2 * PAD)).from_buffer_copy(bytes(PAD) + dct + bytes(PAD))
    cap = sum(sizes) + 64
    out = (C.c_ubyte * cap)()
    n = len(frames)
    oo = (C.c_uint64 * n)(); ol = (C.c_uint64 * n)(); st = (C.c_uint32 * n)()
    want = (C.c_uint64 * n)(*sizes)                                # decompressed_sizes of the batch call, when given
    tot = sim.t_decompress_batch(C.addressof(src), off.ctypes.data, ln.ctypes.data, n, (C.addressof(dbuf) + PAD) if dct else None, len(dct),
                                 n_ctas, warps, take, C.addressof(out), cap, C.addressof(oo), C.addressof(ol), C.addressof(st),
                                 C.addressof(want) if exact_sizes else None, 0, None)
    assert tot >= 0
    return [bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(n)], list(st)


def test_golden_vectors_in_one_batch(sim):
    vecs = helpers.golden_vectors()
    plain = [v for v in vecs if not v[3]]
    outs, st = decompress(sim, [v[1] for v in plain], [len(v[2]) for v in plain])
    for (name, frame, raw, _), got, s in zip(plain, outs, st):
        if frame[4] >> 6 == 0 and not (frame[4] >> 5) & 1:        # no content size in the header: the batch call needs sizes
            assert s == 200, name
        else:
            assert s == 0 and got == raw, name
    withd = [v for v in vecs if v[3]]
    outs, st = decompress(sim, [v[1] for v in withd], [len(v[2]) for v in withd], withd[0][3])
    assert st == [0] * len(withd) and outs == [v[2] for v in withd]


@pytest.mark.parametrize("warps,take,n_ctas", [(8, 32, 1), (8, 32, 2), (7, 16, 1), (8, 3, 2)])
def test_batch_of_small_frames_with_bad_ones(sim, ref, warps, take, n_ctas):
    """70 x 4 KiB level-3 frames (half with checksums) share warps; a corrupted frame, a truncated one and one with a wrong
    checksum get their own status and do not disturb their neighbours."""
    blob, off, ln = corpus.text_segments(70, 4096)
    segs = [bytes(blob[int(o):int(o) + int(l)]) for o, l in zip(off, ln)]
    frames = [ref.compress(s, level=3, checksum=(i % 2 == 0)) for i, s in enumerate(segs)]
    bad = bytearray(frames[10]); bad[len(bad) // 2] ^= 0x10; frames[10] = bytes(bad)       # checksummed: any damage is caught
    frames[21] = frames[21][:-5]
    wrong = bytearray(frames[34]); wrong[-1] ^= 1; frames[34] = bytes(wrong)
    outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=n_ctas, warps=warps, take=take)
    for i, s in enumerate(segs):
        if i in (10, 21, 34):
            assert st[i] != 0, i
        else:
            assert st[i] == 0 and outs[i] == s, i
    assert st[34] == 22                                          # checksum_wrong, from zb_verify_checksums


def test_large_and_multi_block_frames(sim, ref):
    """Frames above the 4 KiB tile take the generic execute kernel; 128 KiB blocks, several blocks per frame, long matches,
    RLE and raw blocks, levels 1..19."""
    text = corpus.text_corpus(1 << 20)
    rng = np.random.default_rng(51)
    segs = [bytes(text[:131072]), bytes(text[50000:50000 + 300000]), bytes(60000), rng.integers(0, 256, 40000).astype(np.uint8).tobytes(),
            (b"abcdefgh" * 9000) + bytes(text[:100]), corpus.binary_blob(70000).tobytes(), bytes(text[3:3 + 5000])]
    frames = [ref.compress(s, level=lv, checksum=True) for s, lv in zip(segs, (3, 3, 1, 3, 19, 7, 3))]
    outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=2, warps=7, take=3)
    assert st == [0] * len(segs) and outs == segs


def test_dictionary_records(sim, ref):
    recs = corpus.json_records(460)
    dct = ref.train_dictionary(16384, recs[:400])
    frames = [ref.compress(r, level=3, dict_data=dct) for r in recs[400:]]
    outs, st = decompress(sim, frames, [len(r) for r in recs[400:]], dct)
    assert st == [0] * 60 and outs == recs[400:]


def test_kernel_to_kernel_round_trip():
    """Frames written by the compression kernels (CPU build) regenerate through the decompression kernels (CPU build)."""
    from tests.test_compress_kernel_host import compress
    csim = dsim = host_encoder.build_sim()
    text = corpus.text_corpus(1 << 20)
    segs = [bytes(text[i * 5000:i * 5000 + 3000 + 97 * i]) for i in range(20)] + [bytes(text[200000:200000 + 140000]), bytes(5000), b"q"]
    frames = compress(csim, segs, checksum=True, n_ctas=3)
    outs, st = decompress(dsim, frames, [len(s) for s in segs], n_ctas=2)
    assert st == [0] * len(segs) and outs == segs


def test_pool_overflow_takes_several_passes(sim, ref):
    """40 frames of 24 KB with 32 frames per warp: their Huffman and FSE tables do not fit one warp's shared-memory pool
    together, so lanes wait for later passes -- same bytes, whatever the pass a lane ran in."""
    text = corpus.text_corpus(1 << 20)
    segs = [bytes(text[i * 20011:i * 20011 + 24000 + 13 * i]) for i in range(40)]
    frames = [ref.compress(s, level=3 + (i % 3), checksum=True) for i, s in enumerate(segs)]
    for warps in (8, 7):
        outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=1, warps=warps, take=32)
        assert st == [0] * len(segs) and outs == segs


def test_batches_with_random_damage_follow_the_reference(sim, ref):
    """A slice of tools/batch_fuzz_decode.py: batches of 64 small frames, a random third corrupted / truncated; healthy
    frames regenerate exactly whatever their warp neighbours do, damaged ones follow the reference."""
    rng = np.random.default_rng(61)
    text = corpus.text_corpus(1 << 20)
    healthy = rejected = 0
    for b in range(4):
        sizes = rng.integers(200, 6000, 64)
        segs = [bytes(text[o:o + int(s)]) for o, s in zip(rng.integers(0, len(text) - 6000, 64), sizes)]
        frames = [ref.compress(s, level=int(rng.integers(1, 6)), checksum=bool(rng.integers(0, 2))) for s in segs]
        bad = set(rng.choice(64, 20, replace=False).tolist())
        for i in bad:
            f = bytearray(frames[i])
            if i % 2:
                f[int(rng.integers(4, len(f)))] ^= 1 << int(rng.integers(0, 8))
            else:
                f = f[:int(rng.integers(5, len(f)))]
            frames[i] = bytes(f)
        outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=1 + b % 2, warps=8 - b % 2, take=(32, 16, 8, 32)[b], exact_sizes=True)
        for i, s in enumerate(segs):
            if i not in bad:
                assert st[i] == 0 and outs[i] == s, (b, i)
                healthy += 1
                continue
            try:                                    # the reference's BATCH path: trailing input after a complete frame is not an error there
                want = ref.batch(False, np.frombuffer(frames[i], dtype=np.uint8), np.zeros(1, dtype=np.uint64),
                                 np.array([len(frames[i])], dtype=np.uint64), dst_len=np.array([len(s)], dtype=np.uint64), threads=1)[0].tobytes()
            except Exception:
                want = None
            if want is None:
                assert st[i] != 0, (b, i)
                rejected += 1
            elif st[i] == 0:
                assert outs[i] == want, (b, i)
    assert healthy == 4 * 44 and rejected > 40


def test_damaged_multi_block_frames_follow_the_reference(sim, ref):
    """Frames of several blocks (in this build anything above 24 KB compressed is scanned by a warp: zb_scan_frames_big /
    zb_scan_blocks_big), half of them damaged in a header, a table description or a payload, or cut short."""
    rng = np.random.default_rng(77)
    text = corpus.text_corpus(2 << 20)
    segs, frames = [], []
    for i in range(10):
        o = int(rng.integers(0, len(text) - 400000)); size = int(rng.integers(140000, 330000))
        s = bytes(text[o:o + size]) if i % 3 else rng.integers(0, 256, size // 3).astype(np.uint8).tobytes() + bytes(text[o:o + size // 2])
        segs.append(s); frames.append(ref.compress(s, level=int(rng.integers(1, 5)), checksum=bool(i & 1)))
    bad = {1, 3, 4, 6, 8}
    for i in bad:
        f = bytearray(frames[i])
        if i % 4 == 0:
            f = f[:int(rng.integers(len(f) // 3, len(f)))]
        else:
            for _ in range(2):
                f[int(rng.integers(6, len(f)))] ^= 1 << int(rng.integers(0, 8))
        frames[i] = bytes(f)
    outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=2, warps=7, take=3, exact_sizes=True)
    rejected = 0
    for i, s in enumerate(segs):
        if i not in bad:
            assert st[i] == 0 and outs[i] == s, i
            continue
        try:
            want = ref.batch(False, np.frombuffer(frames[i], dtype=np.uint8), np.zeros(1, dtype=np.uint64),
                             np.array([len(frames[i])], dtype=np.uint64), dst_len=np.array([len(s)], dtype=np.uint64), threads=1)[0].tobytes()
        except Exception:
            want = None
        if want is None:
            assert st[i] != 0, i
            rejected += 1
        elif st[i] == 0:
            assert outs[i] == want, i
    assert rejected >= 3


def test_content_checksum_of_large_frames(sim, ref):
    """Frames above ZB_XXH_BIG (50 KB in this build, 256 KiB on the device) are hashed by a CTA each (zb_verify_checksums_big):
    every alignment of the frame's start in the output, a length that is not a multiple of 32, and a wrong checksum."""
    text = corpus.text_corpus(1 << 20)
    segs = [bytes(text[100:100 + 3 + 7 * i]) for i in range(5)] + [bytes(text[5000 * i:5000 * i + 60000 + 13 * i]) for i in range(1, 18)]
    frames = [ref.compress(s, level=3, checksum=True) for s in segs]
    bad = bytearray(frames[9]); bad[-2] ^= 0x40; frames[9] = bytes(bad)
    outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=2, warps=7, take=3, exact_sizes=True)
    for i, s in enumerate(segs):
        if i == 9:
            assert st[i] != 0
        else:
            assert st[i] == 0 and outs[i] == s, i
