"""Fuzz of the block-parallel decode path on the CPU build (tests/simt.h): batches of MULTI-BLOCK frames (30 KB - 400 KB,
levels 1-5, with and without checksum, text / incompressible / long runs), a random half damaged (bit flips in headers,
table descriptions and payloads; truncation), through the three mappings the launcher chooses between -- a lane per frame,
a lane per block + tile executor, a lane per block + pointer jumping -- and the warp-cooperative scans and checksums
(this build hands them every frame above 24 KB / 50 KB).  Healthy frames must regenerate exactly; a damaged frame is never
accepted when the reference rejects it, and has the reference's bytes when both accept; all three mappings must agree.
   N=30 SEED=1 python tools/fuzz_multi_block_decode.py
Round 2: N=40 SEED=11 (320 frames x 3 mappings): 160 healthy exact; damaged: 134 rejected by both, 19 accepted by both with equal
bytes, 7 rejected by the kernels alone (the stricter Huffman check, DESIGN section 6).  ASAN build, N=20 SEED=23 and N=6 SEED=5: clean.
   ASAN=1 ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0 LD_PRELOAD=$(gcc -print-file-name=libasan.so) N=10 python tools/fuzz_multi_block_decode.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import corpus
from oracle import RefZstd
from tests import host_encoder
from tests.test_decode_pipeline_host import decompress

if os.environ.get("ASAN") == "1":
    sim = host_encoder.build_sim("/tmp/libzsim_asan.so", ["-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer"])
else:
    sim = host_encoder.build_sim()
ref = RefZstd()
rng = np.random.default_rng(int(os.environ.get("SEED", "1")))
text = corpus.text_corpus(4 << 20)
N = int(os.environ.get("N", "20"))


def ref_one(frame, size):
    try:
        out, _ = ref.batch(False, np.frombuffer(frame, dtype=np.uint8), np.zeros(1, dtype=np.uint64), np.array([len(frame)], dtype=np.uint64),
                           dst_len=np.array([size], dtype=np.uint64), threads=1)
        return out.tobytes()
    except RefZstd.Error:
        return None


def make(kind, size):
    o = int(rng.integers(0, len(text) - size - 1))
    if kind == 0:
        return bytes(text[o:o + size])
    if kind == 1:
        return rng.integers(0, 256, size // 2).astype(np.uint8).tobytes() + bytes(text[o:o + size // 2])
    if kind == 2:
        return bytes(text[o:o + size // 3]) + bytes(size // 3) + bytes([7]) * (size // 3)
    return bytes(text[o:o + 5000]) * (size // 5000)


healthy = rej_both = same = stricter = 0
for it in range(N):
    n = 8
    segs = [make(int(rng.integers(0, 4)), int(rng.integers(30000, 400000))) for _ in range(n)]
    frames = [ref.compress(s, level=int(rng.integers(1, 6)), checksum=bool(rng.integers(0, 2))) for s in segs]
    bad = set(rng.choice(n, n // 2, replace=False).tolist())
    for i in bad:
        f = bytearray(frames[i]); mode = int(rng.integers(0, 4))
        if mode == 0:
            f = f[:int(rng.integers(5, len(f)))]
        elif mode == 1:                                  # somewhere in the first block's headers
            f[int(rng.integers(4, 40))] ^= 1 << int(rng.integers(0, 8))
        else:
            for _ in range(int(rng.integers(1, 4))):
                f[int(rng.integers(4, len(f)))] ^= 1 << int(rng.integers(0, 8))
        frames[i] = bytes(f)
    sizes = [len(s) for s in segs]
    res = []
    for mode in (0, 1, 2):
        sim.t_set_block_path(mode)
        res.append(decompress(sim, frames, sizes, n_ctas=2, warps=7, take=3, exact_sizes=True))
    sim.t_set_block_path(0)
    for i, s in enumerate(segs):
        sts = [r[1][i] for r in res]; outs = [r[0][i] for r in res]
        assert (sts[0] == 0) == (sts[1] == 0) == (sts[2] == 0), ("mappings disagree", it, i, sts)
        if i not in bad:
            assert sts == [0, 0, 0] and outs[0] == outs[1] == outs[2] == s, (it, i, sts)
            healthy += 1
            continue
        want = ref_one(frames[i], len(s))
        if want is None:
            assert sts[0] != 0, ("accepted what the reference rejects", it, i)
            rej_both += 1
        elif sts[0] == 0:
            assert outs[0] == outs[1] == outs[2] == want, (it, i)
            same += 1
        else:
            stricter += 1
    print("iteration %d: healthy %d exact; damaged: %d rejected by both, %d accepted by both with equal bytes, %d rejected by the kernels alone"
          % (it, healthy, rej_both, same, stricter), flush=True)
