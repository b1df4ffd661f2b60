"""tools/gpu_decode_timeline.py reads the idle windows of the batch decode out of a torch.profiler trace; here it reads a
hand-made trace of two steps whose windows are known."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 100


def _tool():
    spec = importlib.util.spec_from_file_location("gpu_decode_timeline", os.path.join(ROOT, "tools", "gpu_decode_timeline.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _k(name, ts, dur):
    return {"ph": "X", "cat": "kernel", "name": "void %s(unsigned int, int*)" % name, "ts": ts, "dur": dur, "args": {}}


def _copy(kind, nbytes, ts, dur, cat="gpu_memcpy"):
    return {"ph": "X", "cat": cat, "name": "Memcpy %s (Device -> Pageable)" % kind, "ts": ts, "dur": dur, "args": {"bytes": nbytes}}


def _step(t, table_copy):
    """One call from its zb_scan_frames at t; its end and the next call's set-up copies, the next scan at t + 1510."""
    ev = [_k("zb_scan_frames", t, 10), _k("zb_place_reduce", t + 10, 5), _k("zb_place_scan", t + 15, 5),
          _copy("DtoH", 48, t + 22, 1),                                   # totals: 2 us after the scan, then 100 us idle
          _k("zb_entropy_decode", t + 123, 400), _k("zb_execute", t + 523, 300), _k("zb_finish", t + 823, 10)]
    if table_copy:
        ev.append(_copy("DtoH", 16 * N, t + 840, 500))
    ev += [_copy("DtoH", 4, t + 1341, 1), _copy("HtoD", 8, t + 1500, 1), _copy("HtoD", 0, t + 1502, 1, cat="gpu_memset")]
    ev.append({"ph": "X", "cat": "user_annotation", "name": "zb200_decompress_batch", "ts": t - 5, "dur": 1350})
    return ev


@pytest.mark.parametrize("table_copy", [True, False])
def test_idle_windows_of_a_known_trace(table_copy):
    tool = _tool()
    ev = _step(0, table_copy) + _step(1510, table_copy) + [_k("zb_scan_frames", 3020, 10)]
    res = tool.analyse({"traceEvents": ev}, N)
    m = res["median"]
    assert res["steps"] == 2
    assert m["period_ms"] == pytest.approx(1.510)
    assert m["place_to_entropy_idle_ms"] == pytest.approx(0.102)
    assert m["seg_table_d2h_ms"] == pytest.approx(0.5 if table_copy else 0.0)
    # from the 4-byte error read-back to the next scan: 158 + 1 + 7 us
    assert m["between_calls_idle_ms"] == pytest.approx(0.166)
    idle = 0.276 if table_copy else 0.276 + 0.5
    assert m["gpu_idle_ms"] == pytest.approx(idle)
    assert m["gpu_busy_ms"] == pytest.approx(1.510 - idle)
    assert m["host_call_ms"] == pytest.approx(1.350)
    gaps = {g["between"]: g["ms"] for g in res["idle_gaps_ms_per_step"]}
    assert gaps["Memcpy DtoH (Device -> Pageable) 48 B -> zb_entropy_decode"] == pytest.approx(0.1)
    assert gaps["Memcpy DtoH (Device -> Pageable) 4 B -> Memcpy HtoD (Device -> Pageable) 8 B"] == pytest.approx(0.158)
