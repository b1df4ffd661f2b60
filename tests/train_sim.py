"""CPU build of the dictionary-training kernels (python_zstandard_b200/csrc/zb_train.cuh) on the SIMT runtime of
tests/simt.h, driven the way zb200_train_dictionary drives them.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess

from tests import host_encoder

TRAIN_SRC = os.path.join(host_encoder.ROOT, "python_zstandard_b200", "csrc", "zb_train.cuh")
LIB = os.path.join(host_encoder.BUILD, "libzt_host.so")

WRAPPERS = r"""
#define ZT_EXPORT extern "C" __attribute__((visibility("default")))
// hash + count of one d (zt_hash_all, zt_count)
static void t_tables(const u8* s, const u64* offs, u32 n_train, u32 f, u32 d, u32 step, std::vector<u32>& hash, std::vector<u32>& freqs)
{
    u32 const n_dmers = (u32)(offs[n_train] - 8 + 1);
    hash.assign(n_dmers, 0); freqs.assign((size_t)1 << f, 0);
    simt::launch(4, 64, [&] { zt_hash_all(s, n_dmers, f, d, hash.data()); });
    simt::launch(4, 64, [&] { zt_count(hash.data(), offs, n_train, step, freqs.data()); });
}
ZT_EXPORT void t_freqs(const u8* s, const u64* offs, u32 n_train, u32 f, u32 d, u32 step, u32* out)
{
    std::vector<u32> hash, freqs; t_tables(s, offs, n_train, f, d, step, hash, freqs);
    memcpy(out, freqs.data(), freqs.size() * 4);
}
// prev[] of every position (zt_prev_local + zt_prev_link)
ZT_EXPORT void t_prev(const u32* hash, u32 n, u32 f, u32* prev)
{
    std::vector<u8> last(n); std::vector<u32> table((size_t)1 << f, 0xFFFFFFFFu);
    simt::launch((n + ZT_CHUNK - 1) / ZT_CHUNK, 128, [&] { zt_prev_local(hash, n, prev, last.data()); });
    simt::launch(1, 128, [&] { zt_prev_link(hash, n, prev, last.data(), table.data()); });
}
// one candidate (k, d) through zt_select: the content lands in dict[*tail .. cap)
ZT_EXPORT void t_select(const u8* s, const u64* offs, u32 n_train, u32 f, u32 d, u32 step, u32 k, u32 cap, u8* dict, u32* tail)
{
    std::vector<u32> hash, freqs; t_tables(s, offs, n_train, f, d, step, hash, freqs);
    u32 const n = (u32)hash.size();
    std::vector<u32> prev(n); t_prev(hash.data(), n, f, prev.data());
    u32 num, esz; zt_epochs(cap, n, k, num, esz);
    std::vector<u32> diff(esz + 2);
    ZtCand cand{k, d, 0, 0};
    ZtSelect A; memset(&A, 0, sizeof A);
    A.samples = s; A.n_dmers[0] = n; A.hash[0] = hash.data(); A.prev[0] = prev.data();
    A.freqs = freqs.data(); A.freqs_stride = 0; A.diff = diff.data(); A.diff_stride = 0; A.dict = dict; A.cap = cap;
    A.tail = tail; A.cand = &cand; A.first = 0;
    simt::launch(1, 128, [&] { zt_select(A); });
}
// zt_entropy + zt_finalize of one content with given statistics (u32[377])
ZT_EXPORT long long t_finalize(const u8* dict, u32 cap, u32 tail, const u32* stats, u32 dict_id, u8* out)
{
    u8 ent[512]; u32 ent_len = 0; long long res = 0;
    simt::launch(1, 32, [&] { zt_entropy(stats, cap - tail, ent, &ent_len); });
    simt::launch(1, 64, [&] { zt_finalize(dict, cap, &tail, ent, &ent_len, dict_id, out, &res); });
    return res;
}
"""


def build():
    """The compression kernel source as tests/host_encoder.py assembles it, then zb_train.cuh up to its launchers.  Built
    with hidden symbols and without unique globals: the same kernels' function-static "shared memory" must not be bound to
    the compression test library's copy when both are loaded in one process."""
    host_encoder.build_compress_sim()
    base = open(os.path.join(host_encoder.BUILD, "zs_host.cpp")).read()
    base = base[:base.index(host_encoder.SIM_WRAPPERS)] if host_encoder.SIM_WRAPPERS in base else base
    tr = open(TRAIN_SRC).read().replace("#pragma once", "")
    tr = tr[:tr.index('extern "C" {')] + "#endif\n"
    text = base + tr + WRAPPERS
    cpp = os.path.join(host_encoder.BUILD, "zt_host.cpp")
    if not (os.path.exists(LIB) and os.path.exists(cpp) and open(cpp).read() == text):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-fvisibility=hidden", "-fvisibility-inlines-hidden", "-fno-gnu-unique", "-I/usr/local/cuda/include", "-o", LIB, cpp])
    L = C.CDLL(LIB)
    vp, u32 = C.c_void_p, C.c_uint32
    L.t_freqs.argtypes = [vp, vp, u32, u32, u32, u32, vp]
    L.t_prev.argtypes = [vp, u32, u32, vp]
    L.t_select.argtypes = [vp, vp, u32, u32, u32, u32, u32, u32, vp, vp]
    L.t_finalize.argtypes = [vp, u32, u32, vp, u32, vp]
    L.t_finalize.restype = C.c_longlong
    return L
