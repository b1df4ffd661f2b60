"""Batch fuzz of ALL decompression kernels on the CPU build (tests/simt.h): batches of 64 small frames in which a random
third is corrupted, truncated or has a wrong checksum.  Healthy frames must regenerate exactly whatever their neighbours
in the warp do; damaged ones must follow the reference (never accepted when it rejects; same bytes when both accept).
   N=200 SEED=1 python tools/batch_fuzz_decode.py        (round 1: 400 batches / 25600 frames against the reference's batch path: 19701 healthy frames exact; damaged:
   4722 rejected by both, 878 accepted by both with equal bytes, 299 rejected by the kernels alone)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import corpus
from oracle import RefZstd
from tests import host_encoder
from tests.test_decode_pipeline_host import decompress

sim = host_encoder.build_sim()
ref = RefZstd()


def ref_batch_one(frame, size):
    """What the reference's BATCH path does with this frame (oracle/ref_batch.c restates decompress_worker,
    c-ext/decompressor.c:1147-1163: one ZSTD_decompressStream call, output size checked, trailing input NOT checked --
    a frame whose checksum flag was flipped off still decodes there, unlike in one-shot ZSTD_decompress)."""
    blob = np.frombuffer(frame, dtype=np.uint8)
    try:
        out, _ = ref.batch(False, blob, np.zeros(1, dtype=np.uint64), np.array([len(frame)], dtype=np.uint64),
                           dst_len=np.array([size], dtype=np.uint64), threads=1)
        return out.tobytes()
    except RefZstd.Error:
        return None


rng = np.random.default_rng(int(os.environ.get("SEED", "1")))
text = corpus.text_corpus(1 << 20)
N = int(os.environ.get("N", "100"))
healthy = damaged_rej = damaged_same = stricter = 0
for b in range(N):
    sizes = rng.integers(200, 6000, 64)
    segs = [bytes(text[o:o + int(s)]) for o, s in zip(rng.integers(0, len(text) - 6000, 64), sizes)]
    frames = [ref.compress(s, level=int(rng.integers(1, 6)), checksum=bool(rng.integers(0, 2))) for s in segs]
    bad = set(rng.choice(64, int(rng.integers(5, 25)), replace=False).tolist())
    for i in bad:
        f = bytearray(frames[i]); kind = int(rng.integers(0, 3))
        if kind == 0: k = int(rng.integers(4, len(f))); f[k] ^= 1 << int(rng.integers(0, 8))
        elif kind == 1: f = f[:int(rng.integers(5, len(f)))]
        else: k = int(rng.integers(4, len(f))); f[k] = int(rng.integers(0, 256))
        frames[i] = bytes(f)
    warps, take = [(8, 32), (7, 16), (8, 8), (8, 32)][b % 4]
    outs, st = decompress(sim, frames, [len(s) for s in segs], n_ctas=1 + b % 2, warps=warps, take=take, exact_sizes=True)
    for i, s in enumerate(segs):
        if i not in bad:
            assert st[i] == 0 and outs[i] == s, (b, i, st[i]); healthy += 1
            continue
        want = ref_batch_one(frames[i], len(s))
        if want is None:
            assert st[i] != 0, (b, i, "accepted what the reference rejects"); damaged_rej += 1
        elif st[i] == 0:
            assert outs[i] == want, (b, i); damaged_same += 1
        else:
            stricter += 1
print("batches", N, "healthy ok", healthy, "| damaged: both reject", damaged_rej, "both accept equal", damaged_same, "kernels stricter", stricter)
