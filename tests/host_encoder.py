"""The CPU build of the kernel source, for the CPU suite.  Test infrastructure only.

build_sim() compiles tests/simt_kernels.cpp with g++: zb_decode.cu and zb_encode.cu as they are, launchers included, on the
mini SIMT runtime of tests/simt.h, with the ctypes wrappers of simt_kernels.cpp.  Those wrappers call the kernels' serial
helpers (FSE normalisation, NCount writer and reader, CTables, Huffman codes and weight headers, decode tables, frame
headers, literal streams) by name, and run the kernels through their launchers.  So every CPU test -- the known-answer
tests against the reference's own FSE_* / HUF_* functions in oracle/_ref included -- checks the source lines the device
runs, from the one library this module builds.
"""
import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "python_zstandard_b200", "csrc")
BUILD = os.path.join(HERE, "_build")
SIM_SRC = os.path.join(HERE, "simt_kernels.cpp")
SIM_LIB = os.path.join(BUILD, "libzsim.so")
# The CPU build of the kernels: simt.h's runtime, the compressor's lock-step markers, and the decoder's big-frame thresholds
# lowered from 512 KiB / 256 KiB so that small test frames reach the warp-cooperative scans and checksums.
SIM_FLAGS = ["-DZB_SIMT_EMULATION", "-DZB_SIMT_STEP()=__syncwarp()", "-DZB_SCAN_BIG=24000u", "-DZB_XXH_BIG=50000u"]


def build_sim(lib=SIM_LIB, extra=()):
    """Host build of the whole kernel source -- zb_decode.cu and zb_encode.cu as they are, launchers included -- on the mini
    SIMT runtime of tests/simt.h, with the wrappers of tests/simt_kernels.cpp.  `extra`: more g++ flags (sanitizers)."""
    import glob
    import hashlib
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    # -Bsymbolic: the library's calls bind to its own definitions -- simt.h's cudaMemsetAsync and the launchers -- even
    # when the process has loaded the CUDA runtime or libzb200.so, which export the same names
    cmd = (["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-Wl,-Bsymbolic", "-I/usr/local/cuda/include", "-I" + CSRC, "-I" + HERE]
           + SIM_FLAGS + list(extra) + [SIM_SRC])
    h = hashlib.sha256(" ".join(cmd).encode())
    for f in sorted(glob.glob(os.path.join(CSRC, "*.cu*"))) + [SIM_SRC, os.path.join(HERE, "simt.h")]:
        h.update(open(f, "rb").read())
    stamp = lib + ".sha256"
    if not (os.path.exists(lib) and os.path.exists(stamp) and open(stamp).read() == h.hexdigest()):
        tmp = "%s.%d.tmp" % (lib, os.getpid())          # processes that build at once each replace the library whole
        subprocess.check_call(cmd + ["-o", tmp])
        os.replace(tmp, lib)
        open(stamp, "w").write(h.hexdigest())
    L = C.CDLL(lib)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
    L.t_any_calls.restype = C.c_ulonglong
    # the serial helpers
    for name in ("t_write_ncount", "t_cost", "t_huf_write_table", "t_huf_cell", "t_read_ncount", "t_frame_header"):
        getattr(L, name).restype = u32
    L.t_frame_header.argtypes = [vp, u64, u32, u32, u32]
    L.t_parse_header.argtypes = [vp, u64, vp]
    # compression, decompression, chains
    L.t_compress_batch.restype = C.c_longlong
    L.t_compress_batch.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, u64, vp, vp, u32, vp, u32, i32, u32]
    L.t_compress_batch2.restype = C.c_longlong
    L.t_compress_batch2.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, u64, vp, vp, i32, u32]
    L.t_compress_chain_run.restype = C.c_longlong
    L.t_compress_chain_run.argtypes = [vp, vp, vp, u32, u32, u32, vp, u64, vp, vp]
    L.t_decode_frame.argtypes = [vp, u64, vp, u32, vp, u64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    L.t_decompress_batch.restype = C.c_longlong
    L.t_decompress_batch.argtypes = [vp, vp, vp, u32, vp, u32, u32, u32, u32, vp, u64, vp, vp, vp, vp, u64, vp]
    L.t_scan_totals.restype = None
    L.t_scan_totals.argtypes = [vp, vp, vp, u32, vp]
    L.t_decompress_chain_run.restype = C.c_longlong
    L.t_decompress_chain_run.argtypes = [vp, vp, vp, u32, C.c_char_p, u64, vp, u64, vp, vp, vp, C.POINTER(C.c_int)]
    # dictionary training
    L.t_freqs.argtypes = [vp, vp, u32, u32, u32, u32, vp]
    L.t_prev.argtypes = [vp, u32, u32, vp]
    L.t_select.argtypes = [vp, vp, u32, u32, u32, u32, u32, u32, vp, vp]
    L.t_finalize.argtypes = [vp, u32, u32, vp, u32, vp]
    L.t_finalize.restype = C.c_longlong
    return L
