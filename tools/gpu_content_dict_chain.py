"""decompress_content_dict_chain on the GPU against the reference's function on one core (tests/chain_ref.py, which is
single-threaded like the reference): revision chains of a 256 KiB text changed by a few seeded 10-200 byte edits per
revision, at 16, 256 and 2048 revisions, and 64 revisions of 8 MiB.  Median of 5 wall times each; the per-kernel profile
and the pointer-doubling rounds of the last GPU call; the card's name and power limit.  Prints one JSON line per chain."""
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


def median_time(fn, reps=5):
    ts = []
    for _ in range(reps):
        t = time.perf_counter(); fn(); ts.append(time.perf_counter() - t)
    return statistics.median(ts)


def main():
    text = corpus.text_corpus().tobytes()
    dctx = zstd.ZstdDecompressor()
    ctx = _native.Context.get(_native.default_device())
    L = _native.lib()
    print(json.dumps({"card": card()}))
    for n, size in [(16, 256 << 10), (256, 256 << 10), (2048, 256 << 10), (64, 8 << 20)]:
        base = (text * (size // len(text) + 1))[:size]
        revs = R.revisions(base, n, seed=n)
        frames = R.compress_chain(revs)
        assert dctx.decompress_content_dict_chain(frames) == revs[-1]
        gpu = median_time(lambda: dctx.decompress_content_dict_chain(frames))
        ref = median_time(lambda: R.decompress_chain(frames))
        L.zb200_profile_enable(ctx.h, 1); L.zb200_profile_reset(ctx.h)
        dctx.decompress_content_dict_chain(frames)
        ms, nl = (C.c_float * 16)(), (C.c_uint32 * 16)()
        L.zb200_profile_read(ctx.h, ms, nl); L.zb200_profile_enable(ctx.h, 0)
        prof = {L.zb200_kernel_name(k).decode(): [round(ms[k], 3), nl[k]] for k in range(16) if nl[k]}
        print(json.dumps({"revisions": n, "fulltext_bytes": size, "compressed_bytes": sum(map(len, frames)),
                          "gpu_s": round(gpu, 5), "ref_1core_s": round(ref, 5), "speedup": round(ref / gpu, 2),
                          "chase_rounds": L.zb200_last_chase_rounds(ctx.h), "kernel_ms_launches": prof}))


if __name__ == "__main__":
    main()
