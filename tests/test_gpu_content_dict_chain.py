"""ZstdDecompressor.decompress_content_dict_chain on the GPU, against the reference's function (tests/chain_ref.py)."""
import os
import random
import re
import struct
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import chain_ref as R                    # noqa: E402
import corpus                            # noqa: E402
import python_zstandard_b200 as zstd     # noqa: E402

pytestmark = pytest.mark.gpu
FRAME_HEADER = b"\x28\xb5\x2f\xfd"


def text(n, off=0):
    return corpus.text_corpus().tobytes()[off:off + n]


def outcome(fn, *a):
    try:
        return "ok", fn(*a)
    except Exception as e:            # (type name, text): ZstdError here is ChainError in the restatement
        return {"ChainError": "ZstdError"}.get(type(e).__name__, type(e).__name__), str(e)


# ---------------------------------------------------------------- the reference's scenarios
def test_bad_inputs_simple():
    dctx = zstd.ZstdDecompressor()
    with pytest.raises(TypeError):
        dctx.decompress_content_dict_chain(b"foo")
    with pytest.raises(TypeError):
        dctx.decompress_content_dict_chain((b"foo", b"bar"))
    with pytest.raises(ValueError, match="^empty input chain$"):
        dctx.decompress_content_dict_chain([])
    with pytest.raises(ValueError, match="^chunk 0 must be bytes$"):
        dctx.decompress_content_dict_chain(["foo"])
    with pytest.raises(ValueError, match="^chunk 0 must be bytes$"):
        dctx.decompress_content_dict_chain([True])
    with pytest.raises(ValueError, match="^chunk 0 is too small to contain a zstd frame$"):
        dctx.decompress_content_dict_chain([FRAME_HEADER])
    with pytest.raises(ValueError, match="^chunk 0 is not a valid zstd frame$"):
        dctx.decompress_content_dict_chain([b"foo" * 8])
    no_size = zstd.ZstdCompressor(write_content_size=False).compress(b"foo" * 64)
    with pytest.raises(ValueError, match="^chunk 0 missing content size in frame$"):
        dctx.decompress_content_dict_chain([no_size])
    frame = zstd.ZstdCompressor().compress(b"foo" * 64)
    frame = frame[0:12] + frame[15:]
    with pytest.raises(zstd.ZstdError, match="^chunk 0 did not decompress full frame$"):
        dctx.decompress_content_dict_chain([frame])


def test_bad_subsequent_input():
    initial = zstd.ZstdCompressor().compress(b"foo" * 64)
    dctx = zstd.ZstdDecompressor()
    with pytest.raises(ValueError, match="^chunk 1 must be bytes$"):
        dctx.decompress_content_dict_chain([initial, "foo"])
    with pytest.raises(ValueError, match="^chunk 1 must be bytes$"):
        dctx.decompress_content_dict_chain([initial, None])
    with pytest.raises(ValueError, match="^chunk 1 is too small to contain a zstd frame$"):
        dctx.decompress_content_dict_chain([initial, FRAME_HEADER])
    with pytest.raises(ValueError, match="^chunk 1 is not a valid zstd frame$"):
        dctx.decompress_content_dict_chain([initial, b"foo" * 8])
    no_size = zstd.ZstdCompressor(write_content_size=False).compress(b"foo" * 64)
    with pytest.raises(ValueError, match="^chunk 1 missing content size in frame$"):
        dctx.decompress_content_dict_chain([initial, no_size])
    frame = zstd.ZstdCompressor(dict_data=zstd.ZstdCompressionDict(b"foo" * 64)).compress(b"bar" * 64)
    frame = frame[0:12] + frame[15:]
    with pytest.raises(zstd.ZstdError, match="^chunk 1 did not decompress full frame$"):
        dctx.decompress_content_dict_chain([initial, frame])


def test_simple():
    original = [b"foo" * 64, b"foobar" * 64, b"baz" * 64, b"foobaz" * 64, b"foobarbaz" * 64]
    chunks = [zstd.ZstdCompressor().compress(original[0])]
    for i, chunk in enumerate(original[1:]):
        chunks.append(zstd.ZstdCompressor(dict_data=zstd.ZstdCompressionDict(original[i])).compress(chunk))
    for i in range(1, len(original)):
        assert zstd.ZstdDecompressor().decompress_content_dict_chain(chunks[0:i]) == original[i - 1]


# ---------------------------------------------------------------- byte parity at real sizes
@pytest.mark.parametrize("n,size,checksum", [(1, 300000, False), (2, 300000, True), (9, 3 * 131072 + 777, True),
                                             (300, 256 << 10, False), (2000, 64 << 10, True)])
def test_revision_chains(n, size, checksum):
    revs = R.revisions(text(size), n, seed=n)
    frames = R.compress_chain(revs, checksum=checksum)
    assert zstd.ZstdDecompressor().decompress_content_dict_chain(frames) == R.decompress_chain(frames) == revs[-1]


def test_chain_written_by_this_package():
    revs = R.revisions(text(400000, 7000), 12, seed=4)
    frames = [zstd.ZstdCompressor().compress(revs[0])]
    for prev, cur in zip(revs, revs[1:]):
        frames.append(zstd.ZstdCompressor(dict_data=zstd.ZstdCompressionDict(prev)).compress(cur))
    assert zstd.ZstdDecompressor().decompress_content_dict_chain(frames) == R.decompress_chain(frames) == revs[-1]


@pytest.mark.parametrize("budget", ["1", "700000", "3000000"])
def test_forced_runs(monkeypatch, budget):
    revs = R.revisions(text(200000, 3000), 24, seed=8)
    frames = R.compress_chain(revs, checksum=True)
    monkeypatch.setenv("ZB200_CHAIN_RUN_BYTES", budget)
    assert zstd.ZstdDecompressor().decompress_content_dict_chain(frames) == revs[-1]
    bad = list(frames)
    b = bytearray(bad[17]); b[-2] ^= 0x10; bad[17] = bytes(b)                # checksum of chunk 17
    assert outcome(zstd.ZstdDecompressor().decompress_content_dict_chain, bad) == outcome(R.decompress_chain, bad)


def test_skippable_and_empty_chunks():
    revs = [text(5000), b"", text(3000, 100), text(3000, 100) + b"more"]
    frames = R.compress_chain(revs)
    assert zstd.ZstdDecompressor().decompress_content_dict_chain(frames) == revs[-1]
    skip = struct.pack("<II", 0x184D2A50, 4) + b"skip"
    for chain in ([frames[0], skip + frames[1]], [frames[0], skip], [frames[0], skip, R.compress_chain([b"", revs[2]])[1]],
                  [frames[0], skip, frames[3]], [skip + b"x"] + frames[1:2]):
        assert outcome(zstd.ZstdDecompressor().decompress_content_dict_chain, chain) == outcome(R.decompress_chain, chain)
    # one skippable chunk: the reference returns the frame's size in uninitialised bytes, this package b""
    assert zstd.ZstdDecompressor().decompress_content_dict_chain([skip]) == b""


def test_first_chunk_with_dict_data():
    samples = [text(2000, 4000 * i) for i in range(400)]
    d = zstd.train_dictionary(8192, samples)
    first = text(50000, 77)
    revs = R.revisions(first, 6, seed=12)
    frames = [zstd.ZstdCompressor(dict_data=d).compress(revs[0])] + R.compress_chain(revs)[1:]
    got = zstd.ZstdDecompressor(dict_data=d).decompress_content_dict_chain(frames)
    assert got == R.decompress_chain(frames, dict_data=d.as_bytes()) == revs[-1]
    assert zstd.ZstdDecompressor(dict_data=d).decompress_content_dict_chain(frames[:1]) == revs[0]
    with pytest.raises(zstd.ZstdError, match="^could not decompress chunk 0: "):
        zstd.ZstdDecompressor().decompress_content_dict_chain(frames)


def test_max_window_size():
    """The reference's stream decoder decodes a frame it holds whole in one pass, and that pass does not check the window
    limit; only a chunk cut short meets it."""
    big = text(2 << 20)
    frames = R.compress_chain([big, big[:-5] + b"abcde"], level=19)
    for mw in (0, 1 << 10, 1 << 20):
        assert (outcome(zstd.ZstdDecompressor(max_window_size=mw).decompress_content_dict_chain, frames)
                == outcome(R.decompress_chain, frames, None, mw))
        cut = [frames[0], frames[1][:-10]]
        assert (outcome(zstd.ZstdDecompressor(max_window_size=mw).decompress_content_dict_chain, cut)
                == outcome(R.decompress_chain, cut, None, mw))


def test_error_order():
    revs = R.revisions(text(30000), 6, seed=2)
    good = R.compress_chain(revs, checksum=True)
    no_size = zstd.ZstdCompressor(write_content_size=False).compress(b"foo" * 64)
    cases = []
    for corrupt in (good[2][:-1] + bytes([good[2][-1] ^ 1]), good[2][:len(good[2]) // 2]):     # bad checksum, cut short
        cases += _order_cases(good, corrupt, no_size)
    for chain in cases:
        want = outcome(R.decompress_chain, chain)
        assert want[0] != "ok"
        assert outcome(zstd.ZstdDecompressor().decompress_content_dict_chain, chain) == want


def _order_cases(good, corrupt, no_size):
    cases = []
    for bad_type in ("str", None, bytearray(good[1])):
        cases += [good[:2] + [corrupt, bad_type] + good[4:], good[:1] + [bad_type, corrupt] + good[3:]]
    cases += [good[:2] + [corrupt, b"foo" * 8] + good[4:], good[:1] + [b"foo" * 8, corrupt] + good[3:],
              good[:2] + [corrupt, no_size], good[:3] + [FRAME_HEADER, corrupt], [corrupt] + good[1:], good[:4] + [corrupt]]
    return cases


def test_mutations():
    revs = R.revisions(text(60000, 9000), 5, seed=6)
    base = R.compress_chain(revs, checksum=True)
    rng = random.Random(17)
    dctx = zstd.ZstdDecompressor()
    for _ in range(60):
        frames = list(base)
        k = rng.randrange(len(frames))
        b = bytearray(frames[k]); b[rng.randrange(len(b))] ^= 1 << rng.randrange(8); frames[k] = bytes(b)
        ref, ours = outcome(R.decompress_chain, frames), outcome(dctx.decompress_content_dict_chain, frames)
        if ref[0] == "ok" and ours[0] != "ok":
            continue                  # a corruption this decoder rejects on every path (tests/test_content_dict_chain_host.py)
        assert ours[0] == ref[0], (ours, ref)
        assert ours == ref if ref[0] == "ok" else re.search(r"chunk (\d+)", ours[1]).group(1) == re.search(r"chunk (\d+)", ref[1]).group(1)
