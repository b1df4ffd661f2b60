"""The lazy mode of the block kernel (explicit greedy / lazy / lazy2 strategy) on the CPU build of the kernel source
(tests/simt_lazy.cpp, built with the flags of tests/host_encoder.py), and the parameter handling that selects it.

Frames go through zb_launch_compress_lazy with the jobs, dictionary and frame window of a real call; each must regenerate
through the reference decoder and the oracle and pass tests/frame_check.py, which holds every offset to the window the
header declares.  The size bars compare against the reference's own libzstd (oracle/_ref) with the same parameters."""
import ctypes as C
import hashlib
import os
import struct

import numpy as np
import pytest

import corpus
from python_zstandard_b200 import compressor as zc
from tests import host_encoder
from tests.frame_check import check_frame

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libzstd_ref.so")
need_ref = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref is built from /root/reference (see oracle/Makefile)")

TEXT = corpus.text_corpus(8 << 20).tobytes()
SILESIA = corpus.silesia_mix(4, 65536)[0][65536:196608].tobytes()    # a json and a binary segment
DEPTH = {zc.STRATEGY_GREEDY: 0, zc.STRATEGY_LAZY: 1, zc.STRATEGY_LAZY2: 2}
ZSTD_c_compressionLevel, ZSTD_c_searchLog, ZSTD_c_minMatch, ZSTD_c_strategy = 100, 104, 105, 107


LAZY_SRC = os.path.join(ROOT, "tests", "simt_lazy.cpp")
LAZY_LIB = os.path.join(host_encoder.BUILD, "libzsim_lazy.so")


def build_lazy_sim():
    """The CPU build of the kernel source with the lazy-mode wrapper (tests/simt_lazy.cpp: simt_kernels.cpp and one more
    function), compiled as tests/host_encoder.py compiles simt_kernels.cpp and rebuilt when a source changes."""
    import glob
    import subprocess
    os.makedirs(host_encoder.BUILD, exist_ok=True)
    cmd = (["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-I/usr/local/cuda/include", "-I" + host_encoder.CSRC,
            "-I" + host_encoder.HERE] + host_encoder.SIM_FLAGS + [LAZY_SRC])
    h = hashlib.sha256(" ".join(cmd).encode())
    for f in sorted(glob.glob(os.path.join(host_encoder.CSRC, "*.cu*"))) + [LAZY_SRC, host_encoder.SIM_SRC,
                                                                             os.path.join(host_encoder.HERE, "simt.h")]:
        h.update(open(f, "rb").read())
    stamp = LAZY_LIB + ".sha256"
    if not (os.path.exists(LAZY_LIB) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest()):
        tmp = "%s.%d.tmp" % (LAZY_LIB, os.getpid())      # processes that build at once each replace the library whole
        subprocess.check_call(cmd + ["-o", tmp])
        os.replace(tmp, LAZY_LIB)
        open(stamp, "w").write(h.hexdigest())
    L = C.CDLL(LAZY_LIB)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    L.t_compress_batch_lazy.restype = C.c_longlong
    L.t_compress_batch_lazy.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, u64, vp, vp, vp, u32, u32, u32, u32, u32]
    L.t_compress_batch.restype = C.c_longlong
    L.t_compress_batch.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, u64, vp, vp, u32, vp, u32, C.c_int, u32]
    return L


@pytest.fixture(scope="module")
def sim():
    return build_lazy_sim()


@pytest.fixture(scope="module")
def ref():
    from oracle import RefZstd
    return RefZstd()


@pytest.fixture(scope="module")
def orc():
    from oracle import Oracle
    return Oracle()


def run(sim, segs, strategy, search_log, min_match, window_log=0, checksum=True, content_size=True, dct=b"", n_ctas=3):
    """[frame] of one batch through the lazy mode.  The segments lie back to back, so a match that reaches in front of
    its frame finds bytes there (and frame_check rejects it)."""
    blob = b"".join(segs) + bytes(64)
    buf = (C.c_ubyte * len(blob)).from_buffer_copy(blob)
    off = np.cumsum([0] + [len(s) for s in segs[:-1]]).astype(np.uint64)
    ln = np.array([len(s) for s in segs], dtype=np.uint64)
    cap = sum(len(s) + len(s) // 128 + 64 for s in segs) + 64
    out = (C.c_ubyte * cap)()
    oo = (C.c_uint64 * len(segs))(); ol = (C.c_uint64 * len(segs))()
    dbuf = (C.c_ubyte * (len(dct) + 64)).from_buffer_copy(dct + bytes(64))
    tot = sim.t_compress_batch_lazy(C.addressof(buf), off.ctypes.data, ln.ctypes.data, len(segs), int(checksum), int(content_size),
                                    n_ctas, C.addressof(out), cap, C.addressof(oo), C.addressof(ol),
                                    C.addressof(dbuf) if dct else None, len(dct), window_log, DEPTH[strategy], search_log, min_match)
    assert tot >= 0 and tot == sum(ol)
    return [bytes(out[oo[i]:oo[i] + ol[i]]) for i in range(len(segs))]


def check(ref, orc, segs, frames, checksum, content_size, dct=b"", dict_id=0):
    for i, (s, f) in enumerate(zip(segs, frames)):
        assert ref.decompress(f, len(s), dct) == s, "segment %d" % i
        assert orc.decompress(f, len(s), dct) == s, "segment %d" % i
        check_frame(f, s, dct, checksum=checksum, content_size=content_size, dict_id=dict_id, oracle=orc)


def ref_size(ref, data, strategy=0, search_log=0, min_match=0, level=3):
    """Bytes of the reference's frame for `data` at `level` with the given match-finder parameters."""
    Z = ref.Z
    c = Z.ZSTD_createCCtx()
    try:
        Z.ZSTD_CCtx_setParameter(c, ZSTD_c_compressionLevel, level)
        for p, v in ((ZSTD_c_strategy, strategy), (ZSTD_c_searchLog, search_log), (ZSTD_c_minMatch, min_match)):
            if v:
                assert not Z.ZSTD_isError(Z.ZSTD_CCtx_setParameter(c, p, v))
        cap = Z.ZSTD_compressBound(len(data))
        out = C.create_string_buffer(cap)
        n = Z.ZSTD_compress2(c, out, cap, data, len(data))
        assert not Z.ZSTD_isError(n)
        return n
    finally:
        Z.ZSTD_freeCCtx(c)


COMBOS = [(s, sl, mm) for s in (zc.STRATEGY_GREEDY, zc.STRATEGY_LAZY, zc.STRATEGY_LAZY2) for sl in (1, 4, 6) for mm in (4, 6)]


@need_ref
@pytest.mark.parametrize("strategy,search_log,min_match", COMBOS)
def test_round_trips(sim, ref, orc, strategy, search_log, min_match):
    """Text, silesia_mix, zeros, random bytes, 1-byte and empty segments; segments of 2^W +- 1 and of several blocks for
    every window log W the blocks are cut differently at; 1 KiB JSON records with a trained dictionary."""
    rng = np.random.default_rng(search_log * 10 + min_match)
    segs = [TEXT[:65536], SILESIA[:65536], SILESIA[65536:], bytes(70000), rng.integers(0, 256, 5000).astype(np.uint8).tobytes(),
            b"x", b"", TEXT[3:3 + 300000]]
    frames = run(sim, segs, strategy, search_log, min_match)
    check(ref, orc, segs, frames, True, True)
    for k, W in enumerate((10, 12, 14, 15, 16, 17)):
        B = 1 << W
        segs = [TEXT[W * 1000:W * 1000 + B - 1], TEXT[W * 2000:W * 2000 + B + 1], TEXT[W * 3000:W * 3000 + 3 * min(B, 1 << 17) + 5]]
        checksum, content_size = k % 2 == 0, k % 3 != 2
        frames = run(sim, segs, strategy, search_log, min_match, window_log=W, checksum=checksum, content_size=content_size)
        check(ref, orc, segs, frames, checksum, content_size)
    dct = open(os.path.join(ROOT, "tests", "golden", "dict.bin"), "rb").read()
    dict_id = struct.unpack_from("<I", dct, 4)[0]
    recs = [r[:1024] for r in corpus.json_records(24)]
    frames = run(sim, recs, strategy, search_log, min_match, dct=dct)
    check(ref, orc, recs, frames, True, True, dct, dict_id)


@pytest.fixture(scope="module")
def text48(sim, ref):
    """48 x 128 KiB text: the lazy mode's sizes (min_match 5) and the reference's at level 3, plain and with the
    lazy2 / search_log 4 / min_match 5 parameters."""
    segs = [TEXT[i * 131072:(i + 1) * 131072] for i in range(48)]
    sizes = {}
    for strategy, sl in ((zc.STRATEGY_GREEDY, 4), (zc.STRATEGY_LAZY, 4), (zc.STRATEGY_LAZY2, 4), (zc.STRATEGY_LAZY2, 2),
                         (zc.STRATEGY_LAZY2, 6)):
        sizes[strategy, sl] = sum(map(len, run(sim, segs, strategy, sl, 5, n_ctas=8)))
    sizes["ref3"] = sum(ref_size(ref, s) for s in segs)
    sizes["ref_lazy2"] = sum(ref_size(ref, s, zc.STRATEGY_LAZY2, 4, 5) for s in segs)
    return sizes


@need_ref
def test_lazy2_size_against_the_reference(text48):
    """lazy2 / search_log 4 / min_match 5 within 3 % of the reference's frames with the same parameters."""
    assert text48[zc.STRATEGY_LAZY2, 4] <= 1.03 * text48["ref_lazy2"], text48


@need_ref
def test_sizes_order_by_strategy_and_depth(text48):
    """Deeper parses and longer chains write smaller frames."""
    s = text48
    assert s[zc.STRATEGY_GREEDY, 4] >= s[zc.STRATEGY_LAZY, 4] >= s[zc.STRATEGY_LAZY2, 4], s
    assert s[zc.STRATEGY_LAZY2, 6] <= s[zc.STRATEGY_LAZY2, 2], s
    assert s[zc.STRATEGY_LAZY2, 4] < s["ref3"], s


@need_ref
def test_small_records_beat_level3(sim, ref):
    """512 x 4 KiB text: lazy2 / search_log 4 smaller than the level-3 kernel on the same batch."""
    segs = [TEXT[i * 4096:(i + 1) * 4096] for i in range(512)]
    lazy = sum(map(len, run(sim, segs, zc.STRATEGY_LAZY2, 4, 5, n_ctas=8)))
    from tests.test_compress_params_host import run as run_level
    level3 = sum(map(len, run_level(sim, segs, 3, 0, False, True, n_ctas=8)))
    assert lazy < level3, (lazy, level3)


# sha256 over the frames of pinned_batch() through lazy2 / search_log 4 / min_match 5, checksum and content size on
PINNED_LAZY2 = "ad40ef0a043eb2ef1acce2260573a26800a0ec12f286de9df2498481785080b9"


def pinned_batch():
    return [TEXT[:200000], TEXT[500000:504096], corpus.json_records(3)[0], bytes(1000), b"ab" * 3000]


@need_ref
def test_pinned_lazy2_frames(sim, ref, orc):
    segs = pinned_batch()
    frames = run(sim, segs, zc.STRATEGY_LAZY2, 4, 5)
    check(ref, orc, segs, frames, True, True)
    assert hashlib.sha256(b"".join(frames)).hexdigest() == PINNED_LAZY2


# ---------------------------------------------------------------- parameters
P = zc.ZstdCompressionParameters


def test_explicit_strategy_is_honoured():
    p = P(strategy=zc.STRATEGY_LAZY2, search_log=4, min_match=5, target_length=16)
    assert (p.strategy, p.search_log, p.min_match, p.target_length) == (5, 4, 5, 16)
    c = zc.ZstdCompressor(compression_params=p)
    cp = c._params()
    assert (cp.strategy, cp.search_log, cp.min_match) == (5, 4, 5)
    q = P.from_level(3, strategy=zc.STRATEGY_GREEDY)
    assert q.strategy == 3 and q.search_log == 1 and q.min_match == 5       # level 3's, reported and used
    cq = zc.ZstdCompressor(compression_params=q)._params()
    assert (cq.strategy, cq.search_log, cq.min_match) == (3, 1, 5)
    assert zc.CParams().strategy == 0 and C.sizeof(zc.CParams) == 32


def test_derived_knobs_stay_reports():
    """from_level fills in the reference's match-finder choice for the level; it never selects the lazy mode."""
    for level in (1, 3, 4, 9, 12, 19):
        p = P.from_level(level)
        cp = zc.ZstdCompressor(compression_params=p)._params()
        assert (cp.strategy, cp.search_log, cp.min_match) == (0, 0, 0)
    p9 = P.from_level(9)
    assert p9.strategy == 5 and p9.search_log > 0
    assert zc.ZstdCompressor(level=9)._params().strategy == 0


@pytest.mark.parametrize("kw,name", [
    (dict(strategy=zc.STRATEGY_FAST), "strategy"), (dict(strategy=zc.STRATEGY_DFAST), "strategy"),
    (dict(strategy=zc.STRATEGY_BTLAZY2), "strategy"), (dict(strategy=zc.STRATEGY_BTULTRA2), "strategy"),
    (dict(search_log=4), "search_log"), (dict(min_match=5), "min_match"), (dict(target_length=8), "target_length"),
    (dict(strategy=zc.STRATEGY_LAZY, hash_log=16), "hash_log"), (dict(strategy=zc.STRATEGY_LAZY2, chain_log=16), "chain_log"),
    (dict(hash_log=16), "hash_log"), (dict(chain_log=16), "chain_log"),
])
def test_refusals(kw, name):
    with pytest.raises(zc.ZstdError, match="compression parameter %s is not supported by the GPU backend" % name):
        P(**kw)
    with pytest.raises(zc.ZstdError, match="compression parameter %s is not supported by the GPU backend" % name):
        P.from_level(3, **kw)


@pytest.mark.parametrize("kw", [dict(strategy=10), dict(strategy=-2), dict(strategy=5, search_log=31), dict(strategy=5, min_match=2),
                                dict(strategy=3, min_match=8), dict(strategy=4, target_length=131073), dict(search_log=-5)])
def test_out_of_range(kw):
    with pytest.raises(zc.ZstdError, match="^unable to set compression context parameter: Parameter is out of bound$"):
        P(**kw)


@need_ref
def test_bounds_and_constants_equal_the_reference(ref):
    """The exported constants, and the bounds they state, are the reference's (ZSTD_cParam_getBounds)."""
    import python_zstandard_b200 as z
    want = dict(STRATEGY_FAST=1, STRATEGY_DFAST=2, STRATEGY_GREEDY=3, STRATEGY_LAZY=4, STRATEGY_LAZY2=5, STRATEGY_BTLAZY2=6,
                STRATEGY_BTOPT=7, STRATEGY_BTULTRA=8, STRATEGY_BTULTRA2=9)
    for k, v in want.items():
        assert getattr(z, k) == v
    Z = ref.Z

    class Bounds(C.Structure):
        _fields_ = [("error", C.c_size_t), ("lower", C.c_int), ("upper", C.c_int)]
    Z.ZSTD_cParam_getBounds.restype = Bounds
    Z.ZSTD_cParam_getBounds.argtypes = [C.c_int]
    for param, lo, hi in ((ZSTD_c_searchLog, z.SEARCHLOG_MIN, z.SEARCHLOG_MAX), (ZSTD_c_minMatch, z.MINMATCH_MIN, z.MINMATCH_MAX),
                          (106, z.TARGETLENGTH_MIN, z.TARGETLENGTH_MAX), (ZSTD_c_strategy, z.STRATEGY_FAST, z.STRATEGY_BTULTRA2)):
        b = Z.ZSTD_cParam_getBounds(param)
        assert (b.lower, b.upper) == (lo, hi), param
