"""zb_execute_tile (frames up to 4 KiB, regenerated in a shared-memory tile with their literals staged in place at the
tile's end) on the CPU build of the kernels (tests/host_encoder.build_decode_sim, lane-per-frame path).

The frames are chosen for the in-place staging: groups whose later literal runs land on an earlier lane's staged
literals, a compressed block without sequences that fills the frame (no margin at all), decompressed sizes larger than
the content, mixed raw / RLE / compressed blocks, every 16-byte phase of the output, short and long offsets on both sides
of the long-match threshold, and dictionary matches that cross into the frame.  Every output must equal the reference's."""
import os

import numpy as np
import pytest

import corpus
from tests import host_encoder
from tests.crafted_frames import _text
from tests.frame_writer import Comp, Dictionary, Frame, Lits, Raw, Rle, write
from tests.test_decode_pipeline_host import decompress

REF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libzstd_ref.so")
pytestmark = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")


@pytest.fixture(scope="module")
def sim():
    L = host_encoder.build_decode_sim()
    L.t_set_block_path(0)
    return L


@pytest.fixture(scope="module")
def orc():
    from oracle import Oracle
    return Oracle()


def _crafted():
    rng = np.random.default_rng(4096)
    out = []
    # zero sequences, literals fill the frame: n_lit == dst_cap, so the block's literals are staged over its own output
    for n in (1, 15, 16, 17, 1000, 4095, 4096):
        out.append(("lits_only_%d" % n, Frame([Comp(Lits(_text(rng, n)), [])]), None))
    out.append(("rle_lits_only", Frame([Comp(Lits(b"q", "rle", regen=4096), [])]), None))
    # the last group of a block: long literal runs in early lanes, the later lanes' runs land on their staged copies
    for ll0 in (40, 100, 300):
        seqs = [(ll0, 3, 3 + 5)] + [(1 + k % 3, 3 + k % 2, 3 + 4 + k) for k in range(40)]
        out.append(("early_long_runs_%d" % ll0, Frame([Comp(Lits(_text(rng, sum(s[0] for s in seqs) + 7)), seqs)]), None))
    # ll = 0 next to long runs, offsets 1..40 and >= 128, lengths 3..4096 across the 32-byte threshold
    seqs, n = [(64, 3, 3 + 64)], 67
    for k, (ml, off) in enumerate([(3, 1), (4, 2), (5, 3), (31, 4), (32, 5), (33, 7), (40, 8), (100, 31), (64, 32),
                                   (65, 33), (200, 40), (3, 128), (500, 130), (31, 200), (32, 333), (1200, 3), (1000, 129)]):
        ll = 0 if k % 2 else 37
        seqs.append((ll, ml, 3 + off))
    lits = _text(rng, sum(s[0] for s in seqs) + 11)
    out.append(("offsets_and_lengths", Frame([Comp(Lits(lits), seqs)]), None))
    out.append(("match_of_4096", Frame([Comp(Lits(b"ab"), [(2, 4094 - 2, 3 + 2)], ), ]), None))
    # several blocks <= 4 KiB: raw, RLE and compressed mixed; raw literals and RLE literals
    out.append(("mixed_blocks", Frame([Raw(_text(rng, 700)), Rle(0x41, 333), Comp(Lits(_text(rng, 90)), [(10, 50, 3 + 600), (30, 40, 3 + 1)]),
                                       Comp(Lits(b"z", "rle", regen=77), [(20, 33, 3 + 1000), (57, 8, 3 + 9)]), Raw(_text(rng, 5))]), None))
    # dictionary matches that straddle the dictionary / output border
    D = Dictionary(_text(rng, 1500), raw=True)
    seqs = [(5, 40, 3 + 20), (0, 8, 3 + 30), (3, 100, 3 + 60), (2, 6, 3 + 1400), (1, 35, 3 + 1530)]
    out.append(("dict_straddle", Frame([Comp(Lits(_text(rng, 30)), seqs)]), D))
    return out


CRAFTED = _crafted()


@pytest.mark.parametrize("extra", [0, 1, 37])
def test_crafted_frames_at_every_phase(sim, orc, extra):
    """Every frame after `k` bytes of padding frames (so the output starts at every phase mod 16), with dst_cap equal
    to the content or `extra` bytes larger (decompressed_sizes given)."""
    for name, F, D in CRAFTED:
        frame, expected, _ = write(F, D)
        dct = D.data if D is not None else b""
        assert orc.decompress(frame, len(expected), dct) == expected, name
        for k in range(0, 16, 5 if extra else 1):
            pad, _, _ = write(Frame([Raw(b"p" * k)]) if k else Frame([Raw(b"")]))
            sizes = [k, len(expected) + extra]
            outs, st = decompress(sim, [pad, frame], sizes, dct, exact_sizes=bool(extra))
            if extra:          # exact sizes: a frame that regenerates less than its decompressed size is an error
                assert st[1] != 0, name
            else:
                assert st == [0, 0] and outs[1] == expected, (name, k)


def test_reference_frames_up_to_4k(sim, orc):
    """Reference-compressed text (Huffman literals staged from the scratch) at several levels and sizes <= 4 KiB,
    decoded as one batch so consecutive frames start at every phase."""
    from oracle import RefZstd
    ref = RefZstd()
    sizes = [1, 3, 17, 100, 1023, 1024, 2047, 4000, 4095, 4096] * 3
    blob, off, ln = corpus.text_segments(len(sizes), 4096)
    raws = [bytes(blob[int(o):int(o) + s]) for o, s in zip(off, sizes)]
    frames = []
    for i, r in enumerate(raws):
        b = np.frombuffer(r, dtype=np.uint8).copy()
        c, cl = ref.batch(True, b, np.array([0], dtype=np.uint64), np.array([len(r)], dtype=np.uint64), level=(1, 3, 19)[i % 3], threads=1)
        frames.append(bytes(c[:int(cl[0])]))
    outs, st = decompress(sim, frames, sizes)
    assert st == [0] * len(frames)
    for f, r, o in zip(frames, raws, outs):
        assert o == r == orc.decompress(f, len(r))
