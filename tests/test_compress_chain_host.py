"""The chain encoder (ZstdCompressor.compress_content_dict_chain) on the CPU: zb_chain_index and the prefix mode of
zb_compress_blocks through tests/simt.h, driven run by run as zb200_compress_chain drives them (tests/chain_encode_sim.py).
Every chain it writes must decode through the reference's chain function (tests/chain_ref.py) and through this package's
chain decoder run on the CPU (tests/chain_sim.py)."""
import hashlib
import mmap
import os
import random
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import chain_encode_sim as E  # noqa: E402
import chain_ref as R          # noqa: E402
import chain_sim as S          # noqa: E402
import corpus                  # noqa: E402

pytestmark = pytest.mark.skipif(not os.path.exists(R.REF), reason="oracle/_ref/libzstd_ref.so not built")


@pytest.fixture(scope="module")
def enc():
    return E.build()


@pytest.fixture(scope="module")
def dec():
    return S.build()


def text(n, off=0):
    return corpus.text_corpus().tobytes()[off:off + n]


def check_round_trip(dec, chunks, frames, every=1):
    """Every prefix decodes to its last chunk through the reference (every `every`-th prefix and the whole chain through the
    CPU build of this package's chain decoder)."""
    assert len(frames) == len(chunks)
    for k in range(len(chunks)):
        assert R.decompress_chain(frames[:k + 1]) == chunks[k], k
        if k % every == 0 or k == len(chunks) - 1:
            assert S.decompress_chain(dec, frames[:k + 1], E.one_run) == chunks[k], k


@pytest.mark.parametrize("n,size", [(1, 1024), (2, 1024), (17, 1024), (64, 1024), (1, 65536), (2, 65536), (17, 65536),
                                    (2, 262144), (2, 300 << 10), (17, 300 << 10)])
def test_revision_chains(enc, dec, n, size):
    revs = R.revisions(text(size), n, seed=n + size)
    frames = E.compress_chain(enc, revs)
    check_round_trip(dec, revs, frames, every=1 if n * size <= (2 << 20) else 4)


def test_size_against_the_reference(enc, dec):
    """64 revisions of 256 KiB: at most 1.15 x the reference's level-3 chain."""
    revs = R.revisions(text(256 << 10), 64, seed=64)
    frames = E.compress_chain(enc, revs)
    ours, ref = sum(map(len, frames)), sum(map(len, R.compress_chain(revs, level=3)))
    assert ours <= 1.15 * ref, (ours, ref)
    check_round_trip(dec, revs, frames, every=16)


def test_frames_hash_to_the_golden_value(enc):
    """The prefix-mode frames do not depend on timing; the GPU test asserts the same digest on the device."""
    frames = E.compress_chain(enc, E.hashed_chain())
    assert hashlib.sha256(b"".join(frames[1:])).hexdigest() == E.GOLDEN_SHA256


def test_output_does_not_depend_on_the_run_cut(enc):
    revs = R.revisions(text(70000, 5000), 9, seed=11)
    want = E.compress_chain(enc, revs)
    for width in (1, 2, 5):
        assert E.compress_chain(enc, revs, run_cut=lambda k, s, w=width: k + w) == want
    assert E.compress_chain(enc, revs, n_ctas=3) == want


@pytest.mark.parametrize("case", sorted(E.shifted_revisions()))
def test_large_shifts_reach_the_whole_predecessor(enc, dec, case):
    chunks = E.shifted_revisions()[case]
    frames = E.compress_chain(enc, chunks)
    check_round_trip(dec, chunks, frames)
    ref = R.compress_chain(chunks, level=3)
    assert len(frames[1]) <= E.shifted_bound(ref[1]), (len(frames[1]), len(ref[1]))


EDGE_CASES = {
    "empty_first": lambda: [b"", text(5000), text(5000, 10)],
    "empty_middle": lambda: [text(5000), b"", text(5000)],
    "empty_last": lambda: [text(5000), text(5000, 7), b""],
    "all_empty": lambda: [b"", b"", b""],
    "short_chunks": lambda: [b"abc", b"abcd", b"abcdefg", b"x", b"abcdefg"],
    "odd_lengths": lambda: [text(4097), text(4099, 1), text(70001, 2), text(70003, 3)],
    "prefix_much_longer": lambda: [text(300000), text(3000, 150000)],
    "prefix_much_shorter": lambda: [text(3000, 150000), text(300000)],
    "edit_at_131071": lambda: [text(262144), text(131071) + b"#" + text(262144)[131072:]],
    "edit_at_131072": lambda: [text(262144), text(131072) + b"#" + text(262144)[131073:]],
}


@pytest.mark.parametrize("case", sorted(EDGE_CASES))
def test_edge_cases(enc, dec, case):
    chunks = EDGE_CASES[case]()
    frames = E.compress_chain(enc, chunks)
    check_round_trip(dec, chunks, frames)


def test_identical_chunks(enc, dec):
    chunks = [text(256 << 10)] * 3
    frames = E.compress_chain(enc, chunks)
    check_round_trip(dec, chunks, frames)
    assert all(len(f) < 64 for f in frames[1:]), [len(f) for f in frames]


def test_unrelated_random_chunks(enc, dec):
    from python_zstandard_b200 import _native
    rng = random.Random(5)
    chunks = [bytes(rng.randrange(256) for _ in range(n)) for n in (200000, 140000, 5)]
    frames = E.compress_chain(enc, chunks)
    check_round_trip(dec, chunks, frames)
    for c, f in zip(chunks[1:], frames[1:]):
        assert len(f) <= _native.lib().zb200_compress_bound(len(c))


def test_checksum(enc, dec):
    revs = R.revisions(text(150000), 4, seed=8)
    frames = E.compress_chain(enc, revs, checksum=True)
    check_round_trip(dec, revs, frames)
    for f in frames:
        assert _frame_info(f).has_checksum == 1


def test_first_chunk_with_a_trained_dictionary(enc):
    d = open(os.path.join(HERE, "golden", "dict.bin"), "rb").read()
    revs = R.revisions(text(20000), 4, seed=2)
    frames = E.compress_chain(enc, revs, dict_data=d)
    for k in range(len(revs)):
        assert R.decompress_chain(frames[:k + 1], dict_data=d) == revs[k]


def _frame_info(f):
    import ctypes as C
    from python_zstandard_b200 import _native
    info = _native.FrameInfo()
    _native.lib().zb200_frame_info(f, len(f), C.byref(info))
    return info


def test_headers(enc):
    revs = [text(100), text(300000, 1), text(70000, 2), b""]
    frames = E.compress_chain(enc, revs)
    for k, f in enumerate(frames):
        info = _frame_info(f)
        assert info.status == 0 and info.content_size == len(revs[k])
        if k:
            assert f[4] & 0x20, "single segment"
            assert info.dict_id == 0 and info.window_size == len(revs[k]) and info.has_checksum == 0


# ---------------------------------------------------------------- the Python layer's argument checks (no device needed)
def test_argument_errors():
    import python_zstandard_b200 as zstd
    c = zstd.ZstdCompressor()
    with pytest.raises(TypeError):
        c.compress_content_dict_chain((b"a", b"b"))
    with pytest.raises(ValueError, match="empty input chain"):
        c.compress_content_dict_chain([])
    with pytest.raises(TypeError, match="item 1 not a bytes like object"):
        c.compress_content_dict_chain([b"a", 5])


def test_far_window_limit():
    """Chunks of ZB_FAR_WINDOW bytes or more (alone or with their predecessor) raise before anything reads them: the 2 GiB
    anonymous mapping is never touched, so no memory is committed."""
    import python_zstandard_b200 as zstd
    c = zstd.ZstdCompressor()
    v = memoryview(mmap.mmap(-1, 2 << 30))
    far = c._FAR_WINDOW
    with pytest.raises(zstd.ZstdError, match="chunk 0"):
        c.compress_content_dict_chain([v[:far]])
    with pytest.raises(zstd.ZstdError, match="chunk 1"):
        c.compress_content_dict_chain([v[:far // 2], v[far // 2:far]])
    with pytest.raises(zstd.ZstdError, match="chunk 2"):
        c.compress_content_dict_chain([b"abc", v[:1 << 30], v[:far - (1 << 30)]])
