"""Wall time of train_dictionary on the device against the reference's fastCover trainer on all host cores.

    python tools/train_dictionary_timing.py [--large]

Sets: the dictionary benchmark's 2000 JSON-like records and, with --large, about 100 MiB of the same records; dictionary
size 112640; default arguments and threads=-1 (82 candidates).  Median of 3 runs each.  Also prints the size of 16384
held-out records compressed by this package with each dictionary, and the GPU's name and power limit."""
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import corpus  # noqa: E402
import python_zstandard_b200 as zstd  # noqa: E402
from tests import train_ref  # noqa: E402


def median_time(fn, runs=3):
    ts, out = [], None
    for _ in range(runs):
        t0 = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t0)
    return statistics.median(ts), out


def main():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", q.stdout.strip(), "| host cores:", os.cpu_count())
    recs = corpus.json_records(2000 + 16384)
    held = recs[2000:]
    sets = [("bench 2000 records", recs[:2000])]
    if "--large" in sys.argv:
        big = corpus.json_records(110000)
        sets.append(("%.0f MiB of records" % (sum(map(len, big)) / 2**20), big))
    zstd.train_dictionary(112640, recs[:2000])            # context creation and first-use costs stay out of the timing
    for name, samples in sets:
        for kw in (dict(), dict(threads=-1)):
            t_gpu, ours = median_time(lambda: zstd.train_dictionary(112640, samples, **kw))
            t_cpu, (theirs, tk, td) = median_time(lambda: train_ref.train_fastcover(112640, samples, nb_threads=os.cpu_count(), **kw))
            sz = {}
            for tag, dct in (("ours", ours), ("ref", zstd.ZstdCompressionDict(theirs))):
                out = zstd.ZstdCompressor(level=3, dict_data=dct).multi_compress_to_buffer(held)
                sz[tag] = sum(len(out[i]) for i in range(len(held)))
            print("%s %s: device %.3f s (k=%d d=%d), reference %.3f s on %d threads (k=%d d=%d); held-out ratio ours %.4f ref %.4f"
                  % (name, kw or "defaults", t_gpu, ours.k, ours.d, t_cpu, os.cpu_count(), tk, td,
                     sum(map(len, held)) / sz["ours"], sum(map(len, held)) / sz["ref"]))


if __name__ == "__main__":
    main()
