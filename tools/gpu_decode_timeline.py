"""Where the GPU idles in the device-resident batch decode: bench.py's `value` loop (262144 x 4 KiB level-3 frames,
zb200_decompress_batch with SRC_DEVICE | DST_DEVICE, the result freed after each call) traced with torch.profiler.

    OUT=/tmp/timeline python tools/gpu_decode_timeline.py               # N=262144 STEPS=10 WARMUP=3 by default
    python tools/gpu_decode_timeline.py --analyse OUT/trace.json         # re-read a trace, no device needed

Two runs in one process: first the loop timed with CUDA events and no profiler (ms per step, as bench.py measures it),
then the same loop under torch.profiler with CUDA activities.  The trace goes to OUT/trace.json, the per-step figures to
OUT/timeline.json.  Per step (a step starts at its zb_scan_frames launch and ends at the next one) it reports:
  place->entropy idle  the GPU idle between the end of zb_place_scan and the start of zb_entropy_decode
  seg table D2H        the device->host copy of the n x 16 B segment table, if the call makes one
  between calls        the GPU idle between the last GPU work of one call and the zb_scan_frames of the next
and every idle gap labelled by the GPU work on either side, so time that goes somewhere else shows up too.
The card's name, power limit and maximum SM clock are read in the same run (nvidia-smi, read-only)."""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GPU_CATS = ("kernel", "gpu_memcpy", "gpu_memset")


def log(*a):
    print(*a, flush=True)


def card_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = "nvidia-smi failed: %r" % (e,)
    return out.splitlines()[0] if out else "unknown"


def label(ev):
    """A stable short name: the kernel's base name, or the copy's kind and size."""
    name = ev.get("name", "")
    if ev.get("cat") == "kernel":
        m = re.search(r"zb_\w+", name)
        return m.group(0) if m else name.split("(")[0][:60]
    b = (ev.get("args") or {}).get("bytes")
    return "%s %s B" % (name, b) if b is not None else name


def analyse(trace, n_frames):
    """Per-step idle windows from a chrome trace written by torch.profiler."""
    evs = [e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") in GPU_CATS]
    evs.sort(key=lambda e: e["ts"])
    starts = [i for i, e in enumerate(evs) if e["cat"] == "kernel" and label(e) == "zb_scan_frames"]
    host = sorted((e for e in trace["traceEvents"] if e.get("ph") == "X" and e.get("cat") == "user_annotation"), key=lambda e: e["ts"])
    steps = []
    for s0, s1 in zip(starts, starts[1:]):
        # the window of a step: from its zb_scan_frames to the next one; the next call's own set-up copies (before its
        # zb_scan_frames) count to this step's "between calls"
        w = evs[s0:s1]
        t0, t1 = w[0]["ts"], evs[s1]["ts"]
        busy, gaps, end = 0.0, [], t0
        prev = w[0]
        for e in w:
            a, b = e["ts"], e["ts"] + e["dur"]
            if a > end:
                gaps.append((label(prev), label(e), a - end, end))
            busy += max(0.0, b - max(a, end))
            if b > end:
                end, prev = b, e
        if t1 > end:
            gaps.append((label(prev), "zb_scan_frames (next call)", t1 - end, end))
        idle = sum(g[2] for g in gaps)

        def find(name):
            for e in w:
                if e["cat"] == "kernel" and label(e) == name:
                    return e
            return None

        place, ent, fin = find("zb_place_scan"), find("zb_entropy_decode"), find("zb_finish")
        p2e = None
        if place and ent:
            lo, hi = place["ts"] + place["dur"], ent["ts"]
            p2e = sum(min(hi, g[3] + g[2]) - max(lo, g[3]) for g in gaps if g[3] < hi and g[3] + g[2] > lo)
        segcopy = [e for e in w if e["cat"] == "gpu_memcpy" and "DtoH" in e.get("name", "")
                   and (e.get("args") or {}).get("bytes", 0) >= 16 * n_frames]
        # between calls: from the last GPU work of this call (its finish or the copies behind it) to the next scan
        last = fin["ts"] + fin["dur"] if fin else None
        if last is not None:
            for e in w:
                if e["ts"] >= last and e["cat"] == "gpu_memcpy" and "DtoH" in e.get("name", ""):
                    last = max(last, e["ts"] + e["dur"])
        between = sum(min(t1, g[3] + g[2]) - max(last, g[3]) for g in gaps if last is not None and g[3] + g[2] > last)
        calls = [h for h in host if h.get("name") == "zb200_decompress_batch" and h["ts"] <= t0]     # the call that launched it
        steps.append({
            "period_ms": (t1 - t0) / 1e3, "gpu_busy_ms": busy / 1e3, "gpu_idle_ms": idle / 1e3,
            "place_to_entropy_idle_ms": None if p2e is None else p2e / 1e3,
            "seg_table_d2h_ms": sum(e["dur"] for e in segcopy) / 1e3,
            "seg_table_d2h": [label(e) for e in segcopy],
            "between_calls_idle_ms": between / 1e3,
            "host_call_ms": calls[-1]["dur"] / 1e3 if calls else None,
            "gaps": [(a, b, d / 1e3) for a, b, d, _ in gaps],
        })
    if not steps:
        raise SystemExit("no complete step in the trace (no two zb_scan_frames launches)")
    med = lambda k: float(np.median([s[k] for s in steps if s[k] is not None])) if any(s[k] is not None for s in steps) else None
    by_gap = {}
    for s in steps:
        for a, b, d in s["gaps"]:
            by_gap.setdefault("%s -> %s" % (a, b), []).append(d)
    gap_table = sorted(((k, float(np.sum(v)) / len(steps), len(v)) for k, v in by_gap.items()), key=lambda x: -x[1])
    kern = {}
    for e in evs[starts[0]:starts[-1]]:
        kern.setdefault(label(e) if e["cat"] == "kernel" else e["cat"], []).append(e["dur"])
    summary = {k: med(k) for k in ("period_ms", "gpu_busy_ms", "gpu_idle_ms", "place_to_entropy_idle_ms", "seg_table_d2h_ms",
                                    "between_calls_idle_ms", "host_call_ms")}
    return {"steps": len(steps), "median": summary,
            "idle_gaps_ms_per_step": [{"between": k, "ms": round(v, 4), "count": c} for k, v, c in gap_table],
            "gpu_work_ms_per_step": {k: round(float(np.sum(v)) / 1e3 / len(steps), 4) for k, v in kern.items()},
            "per_step": [{k: v for k, v in s.items() if k != "gaps"} for s in steps]}


def report(res):
    m = res["median"]
    f = lambda v: "n/a" if v is None else "%.3f" % v
    log("steps traced: %d" % res["steps"])
    log("median per step (ms): period %s, GPU busy %s, GPU idle %s" % (f(m["period_ms"]), f(m["gpu_busy_ms"]), f(m["gpu_idle_ms"])))
    log("  place -> entropy idle   %s" % f(m["place_to_entropy_idle_ms"]))
    log("  segment table D2H       %s" % f(m["seg_table_d2h_ms"]))
    log("  between calls idle      %s" % f(m["between_calls_idle_ms"]))
    log("  host time in the call   %s" % f(m["host_call_ms"]))
    log("idle gaps, mean ms per step:")
    for g in res["idle_gaps_ms_per_step"][:12]:
        log("  %8.4f  %s  (x%d)" % (g["ms"], g["between"], g["count"]))
    log("GPU work, ms per step:", res["gpu_work_ms_per_step"])


def make_batch(n_frames):
    """bench.py's make_batch: n x 4 KiB of S-text compressed by the unmodified reference at level 3."""
    import corpus
    from oracle import RefZstd
    ref = RefZstd()
    blob, off, ln = corpus.text_segments(n_frames, 4096)
    threads = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    cblob, clens = ref.batch(True, blob, off, ln, level=3, threads=threads)
    coff = np.concatenate([[0], np.cumsum(clens)[:-1]]).astype(np.uint64)
    return blob, cblob, coff, clens.astype(np.uint64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--analyse", metavar="TRACE", help="analyse an existing trace instead of running")
    ap.add_argument("--frames", type=int, default=int(os.environ.get("N", "262144")))
    args = ap.parse_args()
    if args.analyse:
        res = analyse(json.load(open(args.analyse)), args.frames)
        report(res)
        return
    out_dir = os.environ.get("OUT") or tempfile.mkdtemp(prefix="zb200_timeline_")
    steps, warmup = int(os.environ.get("STEPS", "10")), int(os.environ.get("WARMUP", "3"))
    n = args.frames
    blob, cblob, coff, clens = make_batch(n)
    log("batch: %d frames, %d B -> %d B" % (n, len(blob), len(cblob)))
    import torch
    from python_zstandard_b200 import _native
    if not torch.cuda.is_available() or _native.device_count() <= 0:
        raise SystemExit("no CUDA device: the timeline is measured on the GPU only")
    card = card_info()
    log("card: %s" % card)
    ctx = _native.Context.get(0)
    L = ctx.L
    stream = torch.cuda.ExternalStream(L.zb200_ctx_stream(ctx.h), device=torch.device("cuda", 0))
    segs = np.stack([coff, clens], axis=1).astype(np.uint64)
    d_src = torch.empty(len(cblob) + 256, dtype=torch.uint8, device="cuda")
    d_src[:len(cblob)].copy_(torch.from_numpy(cblob))
    d_segs = torch.from_numpy(segs.view(np.int64).copy()).cuda()
    torch.cuda.synchronize()

    def step():
        res = C.c_void_p()
        ctx.check(L.zb200_decompress_batch(ctx.h, d_src.data_ptr(), d_segs.data_ptr(), n, None, None,
                                           _native.SRC_DEVICE | _native.DST_DEVICE, C.byref(res)), "zb200_decompress_batch")
        return res

    r = step()
    out = np.empty(len(blob), dtype=np.uint8)
    ctx.check(L.zb200_memcpy_d2h(ctx.h, out.ctypes.data, L.zb200_result_data(r), len(blob)), "d2h")
    L.zb200_result_free(r)
    if not np.array_equal(out, blob):
        raise SystemExit("the batch decoded to different bytes")
    del out
    for _ in range(warmup):
        L.zb200_result_free(step())
    # run 1: CUDA events, no profiler (bench.py's loop, its kernel spans on)
    ctx.profile(True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(stream)
    for _ in range(steps):
        L.zb200_result_free(step())
    e1.record(stream)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    kspans = {k: v[0] / v[1] for k, v in ctx.profile_read().items()}
    log("events: %.3f ms per step = %.1f GB/s; kernel spans (ms per launch): %s"
        % (ms, len(blob) / ms / 1e6, {k: round(v, 3) for k, v in kspans.items()}))
    # run 2: the same loop under torch.profiler
    from torch.profiler import ProfilerActivity, profile, record_function
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps + 1):
            with record_function("zb200_decompress_batch"):
                r = step()
            with record_function("zb200_result_free"):
                L.zb200_result_free(r)
        torch.cuda.synchronize()
    ctx.profile(False)
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "trace.json")
    prof.export_chrome_trace(path)
    res = analyse(json.load(open(path)), n)
    res.update({"card": card, "frames": n, "events_ms_per_step": ms, "events_GBps": len(blob) / ms / 1e6,
                "kernel_spans_ms": kspans, "time": time.strftime("%Y-%m-%d %H:%M:%S")})
    json.dump(res, open(os.path.join(out_dir, "timeline.json"), "w"), indent=1)
    report(res)
    log("trace: %s" % path)


if __name__ == "__main__":
    main()
