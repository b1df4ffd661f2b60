"""Property fuzz of the compression kernels on the CPU build (tests/simt.h): random inputs of many shapes through the
default, two-table and dictionary paths; every frame must regenerate its input through the unmodified reference
decoder and must not exceed the input by more than the format's overhead.
   N=200 SEED=1 python tools/fuzz_compress.py        (round 1: 3 x 500 inputs, 14.5 MB, clean)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import corpus
from oracle import RefZstd
from tests import host_encoder
from tests.test_compress_kernel_host import compress

sim = host_encoder.build_sim()
ref = RefZstd()
rng = np.random.default_rng(int(os.environ.get("SEED", "1")))
text = corpus.text_corpus(1 << 20)
recs = corpus.json_records(500)
dct = ref.train_dictionary(16384, recs[:400])
N = int(os.environ.get("N", "100"))


def sample():
    kind = int(rng.integers(0, 8))
    sizes = [0, 1, 2, 5, 8, 9, 15, 63, 64, 255, 256, 257, 1000, 2047, 2048, 2049, 4096, 9000, 40000, 131071, 131072, 131073]
    w = np.array([3, 3, 3, 3, 3, 3, 3, 5, 5, 5, 5, 5, 10, 6, 6, 6, 8, 6, 4, 1, 2, 1], dtype=np.float64)
    size = int(rng.choice(sizes, p=w / w.sum()))
    if kind == 0: return rng.integers(0, 256, size).astype(np.uint8).tobytes()
    if kind == 1: return rng.integers(0, 4, size).astype(np.uint8).tobytes()
    if kind == 2: return bytes([int(rng.integers(0, 256))]) * size
    if kind == 3:
        pat = rng.integers(0, 256, int(rng.integers(1, 40))).astype(np.uint8).tobytes()
        b = bytearray((pat * (size // len(pat) + 1))[:size])
        for _ in range(size // 97): b[int(rng.integers(0, size))] = int(rng.integers(0, 256))
        return bytes(b)
    if kind == 4: o = int(rng.integers(0, len(text) - size - 1)); return bytes(text[o:o + size])
    if kind == 5: return (recs[int(rng.integers(0, 500))] * (size // 600 + 1))[:size]
    if kind == 6:
        o = int(rng.integers(0, len(text) - size - 1)); h = size // 2
        return bytes(text[o:o + h]) + rng.integers(0, 256, size - h).astype(np.uint8).tobytes()
    return np.clip(rng.normal(128, 3, size), 0, 255).astype(np.uint8).tobytes()


for mode in ("default", "two-table", "dictionary"):
    done = 0; total_in = total_out = 0
    while done < N:
        batch = [sample() for _ in range(int(rng.integers(1, 12)))]
        if not any(batch): continue                                # the API refuses all-empty batches
        frames = compress(sim, batch, checksum=bool(rng.integers(0, 2)), content_size=bool(rng.integers(0, 4)), n_ctas=int(rng.integers(1, 4)),
                          dual=(mode == "two-table"), dct=dct if mode == "dictionary" else b"")
        for s, f in zip(batch, frames):
            back = ref.decompress(f, max(len(s), 1), dct if mode == "dictionary" else b"")
            assert back == s, (mode, len(s))
            assert len(f) <= len(s) + (len(s) >> 7) + 3 * ((len(s) >> 17) + 1) + 18 + 4, (mode, len(s), len(f))
            total_in += len(s); total_out += len(f)
        done += len(batch)
    print("%s: %d inputs, %d -> %d bytes, all regenerate through the reference decoder" % (mode, done, total_in, total_out), flush=True)
