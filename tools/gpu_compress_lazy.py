"""What the lazy-mode knobs cost on the device: device-resident compress GB/s and output size for greedy / lazy / lazy2 at
search_log 2, 4 and 6 (min_match 5) on mixed 128 KiB segments, next to the level-3 and level-4 paths and to the reference's
libzstd with the same parameters on every core of the host, measured in the same run.

    python tools/gpu_compress_lazy.py [--segments N] [--reps R] [--out lazy.json]

GPU rate: input bytes over the wall time of multi_compress_to_buffer on a DeviceBufferWithSegments (input and output on
the device; the call ends in a device synchronise), best of R after a warm-up call.  Sizes are relative to the reference's
level 3 on the same segments."""
import argparse
import concurrent.futures as cf
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ZSTD_c_compressionLevel, ZSTD_c_searchLog, ZSTD_c_minMatch, ZSTD_c_strategy = 100, 104, 105, 107


def ref_all_cores(ref, blob, segs, level, strategy=0, search_log=0, min_match=0):
    """The reference's frames for every segment, one ZSTD_compress2 per segment on a pool of every core (ctypes releases
    the GIL).  Returns (total bytes, seconds)."""
    Z = ref.Z
    local = threading.local()
    mv = memoryview(blob)

    def one(i):
        c = getattr(local, "c", None)
        if c is None:
            c = local.c = Z.ZSTD_createCCtx()
            local.out = C.create_string_buffer(Z.ZSTD_compressBound(1 << 17) + 1024)
        Z.ZSTD_CCtx_reset(c, 2)
        Z.ZSTD_CCtx_setParameter(c, ZSTD_c_compressionLevel, level)
        for p, v in ((ZSTD_c_strategy, strategy), (ZSTD_c_searchLog, search_log), (ZSTD_c_minMatch, min_match)):
            if v:
                Z.ZSTD_CCtx_setParameter(c, p, v)
        o, n = segs[i]
        src = (C.c_char * n).from_buffer(blob, o) if isinstance(blob, bytearray) else mv[o:o + n].tobytes()
        r = Z.ZSTD_compress2(c, local.out, len(local.out), src, n)
        assert not Z.ZSTD_isError(r)
        return r

    t = time.perf_counter()
    with cf.ThreadPoolExecutor(os.cpu_count()) as ex:
        total = sum(ex.map(one, range(len(segs)), chunksize=64))
    return total, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segments", type=int, default=65536)
    ap.add_argument("--size", type=int, default=128 << 10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import corpus
    import python_zstandard_b200 as zstd
    from oracle import RefZstd
    ref = RefZstd()
    ref.Z.ZSTD_CCtx_reset.argtypes = [C.c_void_p, C.c_int]
    ref.Z.ZSTD_CCtx_reset.restype = C.c_size_t
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    card = q[0] if q else "unknown"
    blob_np, off, ln = corpus.silesia_mix(a.segments, a.size)
    blob = bytearray(blob_np.tobytes())
    segs = list(zip(off.tolist(), ln.tolist()))
    table = np.stack([off.astype(np.uint64), ln.astype(np.uint64)], axis=1).tobytes()
    nbytes = int(ln.sum())
    dev = zstd.DeviceBufferWithSegments(torch.frombuffer(blob, dtype=torch.uint8).cuda(), table)
    ref3, _ = ref_all_cores(ref, blob, segs, 3)
    rows = []

    def gpu(params):
        c = zstd.ZstdCompressor(compression_params=params)
        c.multi_compress_to_buffer(dev)                   # warm-up: module load, scratch allocation
        best, size = 1e30, 0
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            res = c.multi_compress_to_buffer(dev)
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t)
            size = res.size                                # bytes of all frames
            del res
        return size, best

    configs = [("level3", dict(compression_level=3), (3, 0, 0, 0)), ("level4", dict(compression_level=4), (4, 0, 0, 0))]
    for name, s in (("greedy", 3), ("lazy", 4), ("lazy2", 5)):
        for sl in (2, 4, 6):
            configs.append(("%s sl%d" % (name, sl), dict(strategy=s, search_log=sl, min_match=5), (3, s, sl, 5)))
    for name, kw, (lvl, s, sl, mm) in configs:
        size, t = gpu(zstd.ZstdCompressionParameters(**kw))
        rsize, rt = ref_all_cores(ref, blob, segs, lvl, s, sl, mm)
        row = dict(config=name, gpu_gbps=nbytes / t / 1e9, gpu_size_vs_ref3=size / ref3,
                   ref_cpu_gbps=nbytes / rt / 1e9, ref_size_vs_ref3=rsize / ref3)
        rows.append(row)
        print("%-10s GPU %7.2f GB/s size %.4f | reference, %d cores: %6.2f GB/s size %.4f"
              % (name, row["gpu_gbps"], row["gpu_size_vs_ref3"], os.cpu_count(), row["ref_cpu_gbps"], row["ref_size_vs_ref3"]), flush=True)
    result = dict(card=card, segments=a.segments, segment_bytes=a.size, cpu_cores=os.cpu_count(), rows=rows)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
