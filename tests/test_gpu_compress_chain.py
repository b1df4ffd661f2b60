"""ZstdCompressor.compress_content_dict_chain on the GPU: every chain it writes decodes through this package's
decompress_content_dict_chain and through the reference's chain function (tests/chain_ref.py)."""
import hashlib
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import chain_encode_sim as E             # noqa: E402
import chain_ref as R                    # noqa: E402
import corpus                            # noqa: E402
import python_zstandard_b200 as zstd     # noqa: E402

pytestmark = pytest.mark.gpu


def text(n, off=0):
    t = corpus.text_corpus().tobytes()
    if off + n > len(t):
        t = t * ((off + n) // len(t) + 1)
    return t[off:off + n]


def check_round_trip(chunks, frames, every=1, dict_data=None, ref=True):
    """Every `every`-th prefix and the whole chain decode to their last chunk through both decoders."""
    assert len(frames) == len(chunks)
    dctx = zstd.ZstdDecompressor(dict_data=dict_data)
    raw = dict_data.as_bytes() if dict_data is not None else None
    for k in range(len(chunks)):
        if k % every and k != len(chunks) - 1:
            continue
        assert dctx.decompress_content_dict_chain(frames[:k + 1]) == chunks[k], k
        if ref:
            assert R.decompress_chain(frames[:k + 1], dict_data=raw, max_window_size=1 << 31) == chunks[k], k


@pytest.mark.parametrize("n,size", [(1, 1024), (2, 1024), (17, 1024), (64, 1024), (2, 65536), (17, 65536), (64, 65536),
                                    (2, 262144), (17, 262144), (2, 300 << 10), (17, 300 << 10), (64, 300 << 10)])
def test_revision_chains(n, size):
    revs = R.revisions(text(size), n, seed=n + size)
    frames = zstd.ZstdCompressor().compress_content_dict_chain(revs)
    check_round_trip(revs, frames)


def test_size_against_the_reference():
    revs = R.revisions(text(256 << 10), 64, seed=64)
    frames = zstd.ZstdCompressor().compress_content_dict_chain(revs)
    ours, ref = sum(map(len, frames)), sum(map(len, R.compress_chain(revs, level=3)))
    assert ours <= 1.15 * ref, (ours, ref)
    check_round_trip(revs, frames, every=8)


def test_device_writes_the_cpu_builds_bytes():
    frames = zstd.ZstdCompressor().compress_content_dict_chain(E.hashed_chain())
    assert hashlib.sha256(b"".join(frames[1:])).hexdigest() == E.GOLDEN_SHA256


@pytest.mark.parametrize("kw", [{}, {"write_checksum": True}, {"write_content_size": False}, {"level": 1}])
def test_first_frame_is_what_compress_writes(kw):
    revs = R.revisions(text(200000), 3, seed=1)
    frames = zstd.ZstdCompressor(**kw).compress_content_dict_chain(revs)
    kw1 = dict(kw, write_content_size=True)
    assert frames[0] == zstd.ZstdCompressor(**kw1).compress(revs[0])
    check_round_trip(revs, frames)


@pytest.mark.parametrize("write_dict_id", [True, False])
def test_first_chunk_with_a_trained_dictionary(write_dict_id):
    d = zstd.ZstdCompressionDict(open(os.path.join(HERE, "golden", "dict.bin"), "rb").read())
    revs = R.revisions(text(30000), 5, seed=2)
    c = zstd.ZstdCompressor(dict_data=d, write_dict_id=write_dict_id)
    frames = c.compress_content_dict_chain(revs)
    assert frames[0] == c.compress(revs[0])
    check_round_trip(revs, frames, dict_data=d)


def test_headers_and_checksums():
    import ctypes as C
    from python_zstandard_b200 import _native
    revs = [text(100), text(300000, 1), text(70000, 2), b""]
    frames = zstd.ZstdCompressor(write_checksum=True).compress_content_dict_chain(revs)
    for k, f in enumerate(frames):
        info = _native.FrameInfo()
        _native.lib().zb200_frame_info(f, len(f), C.byref(info))
        assert info.status == 0 and info.content_size == len(revs[k]) and info.has_checksum == 1
        if k:
            assert f[4] & 0x20 and info.dict_id == 0 and info.window_size == len(revs[k])
    check_round_trip(revs, frames)


def test_edge_cases():
    import random
    rng = random.Random(5)
    base = text(262144)
    cases = [
        [b"", text(5000), text(5000, 10)], [text(5000), b"", text(5000)], [text(5000), text(5000, 7), b""], [b"", b"", b""],
        [b"abc", b"abcd", b"abcdefg", b"x", b"abcdefg"], [text(4097), text(4099, 1), text(70001, 2), text(70003, 3)],
        [text(300000), text(3000, 150000)], [text(3000, 150000), text(300000)],
        [base, base[:131071] + b"#" + base[131072:]], [base, base[:131072] + b"#" + base[131073:]],
    ]
    for chunks in cases:
        check_round_trip(chunks, zstd.ZstdCompressor().compress_content_dict_chain(chunks))
    same = [base] * 3
    frames = zstd.ZstdCompressor().compress_content_dict_chain(same)
    check_round_trip(same, frames)
    assert all(len(f) < 64 for f in frames[1:]), [len(f) for f in frames]
    rnd = [bytes(rng.randrange(256) for _ in range(n)) for n in (200000, 140000, 5)]
    frames = zstd.ZstdCompressor().compress_content_dict_chain(rnd)
    check_round_trip(rnd, frames)
    from python_zstandard_b200 import _native
    assert all(len(f) <= _native.lib().zb200_compress_bound(len(c)) for c, f in zip(rnd[1:], frames[1:]))


def test_2000_revisions():
    revs = R.revisions(text(256 << 10), 2000, seed=2000)
    frames = zstd.ZstdCompressor().compress_content_dict_chain(revs)
    check_round_trip(revs, frames, every=250)


def test_8mib_revisions_reach_beyond_the_reference_window():
    """The reference at level 3 reaches 2 MiB back; chunk k here reaches all of chunk k - 1."""
    revs = R.revisions(text(8 << 20), 4, seed=8)
    frames = zstd.ZstdCompressor().compress_content_dict_chain(revs)
    check_round_trip(revs, frames)
    assert sum(map(len, frames)) < sum(map(len, R.compress_chain(revs, level=3)))


@pytest.mark.parametrize("case", sorted(E.shifted_revisions()))
def test_large_shifts_reach_the_whole_predecessor(case):
    chunks = E.shifted_revisions()[case]
    frames = zstd.ZstdCompressor().compress_content_dict_chain(chunks)
    check_round_trip(chunks, frames)
    ref = R.compress_chain(chunks, level=3)
    assert len(frames[1]) <= E.shifted_bound(ref[1]), (len(frames[1]), len(ref[1]))


def test_300mib_chunks_use_offset_code_28():
    """Offsets of ~300 MiB, between 2^28 and 2^29: OF code 28, the last one the predefined distribution covers.  The corpus
    repeats every 8 MiB, but the first 8 MiB of the second chunk have no earlier copy in that chunk: the frame stays under
    1 MiB only if they are matched ~300 MiB back."""
    base = text(300 << 20)
    revs = R.revisions(base, 2, seed=300)
    del base
    frames = zstd.ZstdCompressor().compress_content_dict_chain(revs)
    assert len(frames[1]) < (1 << 20), len(frames[1])
    assert zstd.ZstdDecompressor().decompress_content_dict_chain(frames) == revs[1]
    assert R.decompress_chain(frames, max_window_size=1 << 31) == revs[1]


@pytest.mark.parametrize("budget", ["1", "700000", "3000000"])
def test_forced_runs(monkeypatch, budget):
    revs = R.revisions(text(300000), 9, seed=12)
    want = zstd.ZstdCompressor(write_checksum=True).compress_content_dict_chain(revs)
    monkeypatch.setenv("ZB200_CHAIN_RUN_BYTES", budget)
    assert zstd.ZstdCompressor(write_checksum=True).compress_content_dict_chain(revs) == want
    check_round_trip(revs, want, every=4)


def test_600mib_chunks_use_offset_code_29():
    """Offsets of ~600 MiB > 2^29: OF code 29, which the predefined distribution does not cover, so every block that uses it
    must carry a compressed (or flat) OF table.  As above, the frame stays under 1 MiB only if the second chunk's first 8 MiB
    are matched ~600 MiB back."""
    base = text(600 << 20)
    revs = R.revisions(base, 2, seed=600)
    del base
    frames = zstd.ZstdCompressor().compress_content_dict_chain(revs)
    assert len(frames[1]) < (1 << 20), len(frames[1])
    assert zstd.ZstdDecompressor().decompress_content_dict_chain(frames) == revs[1]
    assert R.decompress_chain(frames, max_window_size=1 << 31) == revs[1]
