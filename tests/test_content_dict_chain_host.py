"""Chain mode of the block-parallel decode (decompress_content_dict_chain) on the CPU: the kernels through tests/simt.h,
driven run by run as zb200_decompress_chain drives them (tests/chain_sim.py), against the reference's function over ctypes
(tests/chain_ref.py)."""
import os
import random
import struct
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import chain_ref as R          # noqa: E402
import chain_sim as S          # noqa: E402
import corpus                  # noqa: E402
import frame_writer as fw      # noqa: E402
import host_encoder            # noqa: E402

pytestmark = pytest.mark.skipif(not os.path.exists(R.REF), reason="oracle/_ref/libzstd_ref.so not built")


@pytest.fixture(scope="module")
def sim():
    return host_encoder.build_sim()


def one_run(k, sizes):
    return len(sizes)


def text(n, off=0):
    return corpus.text_corpus().tobytes()[off:off + n]


def ref_outcome(frames):
    """('ok', bytes) or ('err', chunk index) of the reference."""
    try:
        return "ok", R.decompress_chain(frames)
    except (ValueError, R.ChainError) as e:
        import re
        return "err", int(re.search(r"chunk (\d+)", str(e)).group(1))


def sim_outcome(sim, frames, cut=one_run):
    try:
        return "ok", S.decompress_chain(sim, frames, cut)
    except S.ChainSimError as e:
        return "err", e.chunk


@pytest.mark.parametrize("n,checksum", [(1, False), (2, True), (9, False), (9, True), (300, False)])
def test_revision_chains(sim, n, checksum):
    size = 40000 if n == 300 else 3 * 131072 + 777           # several 128 KiB blocks, except for the long chain
    revs = R.revisions(text(size), n, seed=n)
    frames = R.compress_chain(revs, checksum=checksum)
    assert S.decompress_chain(sim, frames, one_run) == R.decompress_chain(frames) == revs[-1]


def test_every_run_cut(sim):
    revs = R.revisions(text(70000, 1000), 9, seed=5)
    frames = R.compress_chain(revs, checksum=True)
    want = R.decompress_chain(frames)
    for width in range(1, 10):
        assert S.decompress_chain(sim, frames, lambda k, s, w=width: k + w) == want
    rng = random.Random(2)
    for _ in range(6):           # uneven runs
        cuts = sorted(rng.sample(range(1, 9), rng.randint(1, 4)))
        assert S.decompress_chain(sim, frames, lambda k, s: next((c for c in cuts if c > k), len(s))) == want


# ---------------------------------------------------------------- hand-built frames (tests/frame_writer.py)
PREV = b"".join(b"revision %04d; " % i for i in range(300))


def crafted(F):
    """The chain [PREV compressed, F written with PREV as a raw-content prefix]."""
    data, expected, _ = fw.write(F, fw.Dictionary(PREV, raw=True))
    return [R.compress_chain([PREV])[0], data], expected


def check_both(sim, frames, expect_ok):
    ref, ours = ref_outcome(frames), sim_outcome(sim, frames)
    assert ours == ref, (ours[0], ref[0])
    assert (ref[0] == "ok") == expect_ok


def test_match_reaches_exactly_the_first_prefix_byte(sim):
    lits = b"0123456789"
    F = fw.Frame([fw.Comp(fw.Lits(lits), [(10, 20, 10 + len(PREV) + 3)])], single_segment=True)
    frames, expected = crafted(F)
    assert expected == lits + PREV[:20]
    check_both(sim, frames, True)


def test_match_one_byte_before_the_prefix_is_rejected(sim):
    F = fw.Frame([fw.Comp(fw.Lits(b"0123456789"), [(10, 20, 10 + len(PREV) + 1 + 3)])], single_segment=True)
    frames, expected = crafted(F)
    assert expected is None
    check_both(sim, frames, False)
    assert sim_outcome(sim, frames)[1] == 1


@pytest.mark.parametrize("ll,ov", [(0, 1), (2, 2), (3, 3)])
def test_repcode_in_the_first_sequence_reaches_into_the_prefix(sim, ll, ov):
    F = fw.Frame([fw.Comp(fw.Lits(b"xyz"[:ll] + b"tail"), [(ll, 6, ov)])], single_segment=True)
    frames, expected = crafted(F)
    assert expected is not None
    check_both(sim, frames, True)


def test_repeat_table_in_a_prefixed_chunk_is_rejected(sim):
    F = fw.Frame([fw.Comp(fw.Lits(b"abcdefgh"), [(8, 5, 3 + 100)], ll=fw.Table("rep", fallback=fw.RLE_T(8)))], single_segment=True)
    frames, expected = crafted(F)
    assert expected is None
    check_both(sim, frames, False)


def test_treeless_literals_in_a_prefixed_chunk_are_rejected(sim):
    F = fw.Frame([fw.Comp(fw.Lits(b"abcabcab" * 4, mode="treeless", weights=[0] * 97 + [1, 1, 2]), [])], single_segment=True)
    frames, expected = crafted(F)
    assert expected is None
    check_both(sim, frames, False)


def test_dictionary_id_in_a_prefixed_chunk_is_rejected(sim):
    F = fw.Frame([fw.Comp(fw.Lits(b"abc"), [(3, 10, 3 + 50)])], dict_id=5)
    frames, _ = crafted(F)
    check_both(sim, frames, False)
    assert sim_outcome(sim, frames) == ("err", 1)
    with pytest.raises(R.ChainError, match="chunk 1: Dictionary mismatch"):
        R.decompress_chain(frames)


def test_empty_fulltext_mid_chain(sim):
    revs = [text(5000), b"", text(3000, 100), text(3000, 100) + b"more"]
    frames = R.compress_chain(revs)
    check_both(sim, frames, True)
    assert sim_outcome(sim, frames)[1] == revs[-1]


def test_chunk_that_starts_with_a_skippable_frame(sim):
    """The reference's stream decoder stops behind the skippable frame: the chunk's fulltext is empty, so the chunk
    after it has an empty prefix."""
    revs = R.revisions(text(6000), 3, seed=9)
    frames = R.compress_chain(revs)
    skip = struct.pack("<II", 0x184D2A50, 4) + b"skip"
    assert R.decompress_chain([frames[0], skip + frames[1]]) == b""
    check_both(sim, [frames[0], skip + frames[1]], True)
    check_both(sim, [frames[0], skip], True)
    after = R.compress_chain([b"", revs[2]])[1]
    check_both(sim, [frames[0], skip, after], True)
    assert sim_outcome(sim, [frames[0], skip, frames[2]]) == ref_outcome([frames[0], skip, frames[2]])


def test_mutations(sim):
    """300 single-bit flips of a 4-chunk chain: never accept what the reference rejects, reject at the same chunk, and
    give the same bytes when both accept.  Some flips make the reference decode other bytes (no checksum) where this
    decoder rejects the chunk: the reference's Huffman fast loop does not check that a literal stream is consumed exactly
    (DESIGN.md section 6), and the batch paths reject those frames the same way."""
    revs = R.revisions(text(9000, 20000), 4, seed=1)
    base = R.compress_chain(revs, checksum=False)
    rng = random.Random(300)
    stricter = 0
    for _ in range(300):
        frames = list(base)
        k = rng.randrange(len(frames))
        b = bytearray(frames[k])
        i = rng.randrange(len(b))
        b[i] ^= 1 << rng.randrange(8)
        frames[k] = bytes(b)
        ref, ours = ref_outcome(frames), sim_outcome(sim, frames)
        if ref[0] == "err":
            assert ours == ref, (k, i)
        elif ours[0] == "err":
            stricter += 1
        else:
            assert ours == ref, (k, i)
    assert stricter <= 30
