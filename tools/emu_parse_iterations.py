"""Parse-loop iterations per record on the CPU build of the compression kernel (tests/simt.h counts the votes that drive
the loop): the 256-byte-unit instantiation that calls with only small blocks get, against the 1024-byte one.
   python tools/emu_parse_iterations.py"""
import ctypes as C, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import host_encoder
from tests.test_compress_kernel_host import compress
from oracle import RefZstd
import corpus

ref = RefZstd()
recs = corpus.json_records(560)
dct = ref.train_dictionary(16384, recs[:400])
sample = recs[400:]


def build(tag, extra):
    host_encoder.build_compress_sim()
    cpp = os.path.join(host_encoder.BUILD, "zs_host.cpp"); lib = "/tmp/libzs_iter_%s.so" % tag
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-I/usr/local/cuda/include"] + extra + ["-o", lib, cpp])
    L = C.CDLL(lib); L.t_compress_batch.restype = C.c_longlong; L.t_any_calls.restype = C.c_ulonglong
    L.t_compress_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                   C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_uint32]
    return L


for tag, extra in (("unit1024", ["-DZE_SMALL_MAX=0"]), ("unit256", [])):
    L = build(tag, extra)
    L.t_any_calls(1)
    frames = compress(L, sample, n_ctas=1, dct=dct)
    calls = L.t_any_calls(1)
    size = sum(map(len, frames))
    print("%s: %.0f loop votes per record (parse iterations + a few from the link phase), %d bytes" % (tag, calls / len(sample), size))
