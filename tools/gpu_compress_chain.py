"""compress_content_dict_chain on the GPU against the reference's chain writer on one core (tests/chain_ref.py:compress_chain,
one ZSTD_CCtx_refPrefix + ZSTD_compress2 per revision at level 3): revision chains of a 256 KiB text changed by a few seeded
10-200 byte edits per revision, at 16, 256 and 2048 revisions, and 64 revisions of 8 MiB.  Median of 5 wall times for the
GPU, of 3 for the reference; both totals in bytes; the per-kernel profile of one GPU call; the card's name and power limit.
The round trip (this package's chain decoder) is checked outside the timed region.  Prints one JSON line per chain."""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import chain_ref as R                    # noqa: E402
import corpus                            # noqa: E402
import python_zstandard_b200 as zstd     # noqa: E402
from python_zstandard_b200 import _native  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        return q.stdout.strip().splitlines()[0]
    except (OSError, IndexError):
        return "unknown"


def median_time(fn, reps):
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); fn(); ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def main():
    text = corpus.text_corpus().tobytes()
    cctx, dctx = zstd.ZstdCompressor(), zstd.ZstdDecompressor()
    ctx = _native.Context.get(_native.default_device())
    L = _native.lib()
    print(json.dumps({"card": card()}))
    for n, size in [(16, 256 << 10), (256, 256 << 10), (2048, 256 << 10), (64, 8 << 20)]:
        base = (text * (size // len(text) + 1))[:size]
        revs = R.revisions(base, n, seed=n)
        frames = cctx.compress_content_dict_chain(revs)
        assert dctx.decompress_content_dict_chain(frames) == revs[-1]
        assert dctx.decompress_content_dict_chain(frames[:n // 2]) == revs[n // 2 - 1]
        ref_frames = R.compress_chain(revs)
        gpu = median_time(lambda: cctx.compress_content_dict_chain(revs), 5)
        ref = median_time(lambda: R.compress_chain(revs), 3)
        L.zb200_profile_enable(ctx.h, 1); L.zb200_profile_reset(ctx.h)
        cctx.compress_content_dict_chain(revs)
        ms, nl = (C.c_float * 16)(), (C.c_uint32 * 16)()
        L.zb200_profile_read(ctx.h, ms, nl); L.zb200_profile_enable(ctx.h, 0)
        prof = {L.zb200_kernel_name(k).decode(): [round(ms[k], 3), nl[k]] for k in range(16) if nl[k]}
        print(json.dumps({"revisions": n, "fulltext_bytes": size, "gpu_bytes": sum(map(len, frames)),
                          "ref_bytes": sum(map(len, ref_frames)), "gpu_s": round(gpu, 5), "ref_1core_s": round(ref, 5),
                          "kernel_ms_launches": prof}))


if __name__ == "__main__":
    main()
