"""The chain encoder (compress_content_dict_chain) on the CPU: zb_chain_index and the prefix mode of zb_compress_blocks from
zb_encode.cu on tests/simt.h (the same host build host_encoder.build_compress_sim makes), then the frame layout kernels,
driven run by run as zb200_compress_chain (zb_api.cu) drives them on the device.  Chunk 0 goes through the CPU build of the
batch path (host_encoder's t_compress_batch), as the launcher sends it through zb200_compress_batch_ptrs.
TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

import host_encoder as H

LIB = os.path.join(H.BUILD, "libzc_chain_sim.so")

# SHA-256 over frames 1.. of HASHED_CHAIN (the prefix-mode frames): the device and the CPU build must write these very bytes
GOLDEN_SHA256 = "148c76f2f6c1ec979e55c543bece7b967e6c1c59245a97c60294e9fd20b41235"


def hashed_chain():
    """The chain whose frames GOLDEN_SHA256 pins: 5 seeded revisions of 40000 bytes of the text corpus."""
    import chain_ref
    import corpus
    return chain_ref.revisions(corpus.text_corpus().tobytes()[3000:43000], 5, seed=3)


def shifted_revisions():
    """{name: [A, B]}: B is A (256 KiB of the text corpus) with 2-20 KB inserted, deleted or moved, at the front or in the
    middle -- far more than the few hundred bytes chain_ref.revisions shifts, so the bytes of B sit far from their place
    in A.  Frame 1 of each must cost about what the reference's refPrefix loop pays, not what B costs on its own."""
    import corpus
    t = corpus.text_corpus().tobytes()
    A, X = t[:256 << 10], t[1 << 20:(1 << 20) + 40000]
    return {"insert_2k_front": [A, X[:2000] + A], "insert_12k_front": [A, X[:12000] + A],
            "insert_16k_middle": [A, A[:100000] + X[:16384] + A[100000:]], "delete_12k_front": [A, A[12000:]],
            "delete_20k_middle": [A, A[:90000] + A[110000:]], "move_20k_front_to_middle": [A, A[20000:150000] + A[:20000] + A[150000:]]}


def shifted_bound(ref_frame):
    """What frame 1 of a shifted_revisions() chain may cost against the reference's frame 1 (at least a 3 x margin below
    compressing B alone, which costs ~70-90 KB)."""
    return 1.5 * len(ref_frame) + 512


WRAPPERS = r"""
static u32 t_chain_log(u64 len)          // as zb200_compress_chain sizes a chunk's index: two keys per sampled position at a load <= 1/2, at least 16 slots
{
    u64 const npos = len >= 8 ? (len - 8) / ZE_CHAIN_STEP + 1 : 0;
    u32 L = 4; while ((1ull << L) < 4 * npos) L++;
    return L;
}
// One run: chunk 0 of the run is the prefix of chunk 1 only; chunks 1..m-1 become frames.  src holds the run's chunks back to
// back (slack in front and behind), seg_off / seg_len locate them.  Returns the frames' total bytes.
extern "C" long long t_compress_chain_run(const u8* src, const u64* seg_off, const u64* seg_len, u32 m, u32 checksum, u32 n_ctas,
                                          u8* out, u64 out_cap, u64* out_off, u64* out_len)
{
    std::vector<u64> tab_off(m + 1, 0), pos_off(m + 1, 0); std::vector<u32> logs(m);
    for (u32 s = 0; s < m; s++) {
        logs[s] = t_chain_log(seg_len[s]);
        tab_off[s + 1] = tab_off[s] + (1ull << logs[s]);
        pos_off[s + 1] = pos_off[s] + (seg_len[s] >= 8 ? (seg_len[s] - 8) / ZE_CHAIN_STEP + 1 : 0);
    }
    std::vector<u32> tabs(tab_off[m], 0xFFFFFFFFu);
    std::vector<ZeChainSeg> cs(m);
    for (u32 s = 0; s < m; s++) {
        cs[s].start = seg_off[s]; cs[s].tab = tabs.data() + tab_off[s]; cs[s].log = logs[s]; cs[s].len = (u32)seg_len[s];
        cs[s].prev_tab = s ? tabs.data() + tab_off[s - 1] : nullptr; cs[s].prev_log = s ? logs[s - 1] : 0; cs[s].prev_len = s ? (u32)seg_len[s - 1] : 0;
    }
    if (pos_off[m]) simt::launch(4, 256, [&] { zb_chain_index(src, cs.data(), pos_off.data(), m); });
    u32 const nf = m - 1;
    std::vector<ZbSegment> segs(nf); std::vector<ZeBlockJob> jobs; std::vector<ZeSegInfo> info(nf);
    for (u32 f = 0; f < nf; f++) {
        u32 const s = f + 1;
        segs[f].offset = seg_off[s]; segs[f].length = seg_len[s];
        info[f].first_job = jobs.size(); info[f].n_jobs = 0; info[f].pad = 0;
        for (u64 pos = 0; pos < seg_len[s];) {
            u32 const sz = (u32)(seg_len[s] - pos < ZE_BLOCK ? seg_len[s] - pos : ZE_BLOCK);
            ZeBlockJob j; j.src_pos = seg_off[s] + pos; j.size = sz; j.seg = s; j.first = pos == 0; j.last = pos + sz == seg_len[s];
            jobs.push_back(j); info[f].n_jobs++; pos += sz;
        }
    }
    u32 const nj = (u32)jobs.size();
    u64 const slot_bytes = ((u64)ZE_BLOCK + (ZE_BLOCK >> 7) + 64 + 15) & ~15ull;
    std::vector<u8> slots((size_t)(nj + 1) * slot_bytes); std::vector<ZeBlockOut> outs(nj + 1);
    if (n_ctas > nj) n_ctas = nj ? nj : 1;
    ZePScratch* scratch = (ZePScratch*)aligned_alloc(64, ((sizeof(ZePScratch) + 63) & ~(size_t)63) * n_ctas);
    u32 counter = 0;
    ZeDict dict; memset(&dict, 0, sizeof dict); dict.cct = cs.data();
    ZeUpload up; up.progress = nullptr; up.total = 0; up.status = nullptr;
    if (nj) simt::launch(n_ctas, ZE_THREADS, [&] { zb_compress_blocks<false, ZE_UNIT, false, true>(src, jobs.data(), nj, (ZeScratch*)scratch, slots.data(), slot_bytes, outs.data(), &counter, dict, up); });
    free(scratch);
    ZeParams P; P.checksum = checksum; P.content_size = 1; P.dict_id = 0; P.level = 3; P.window_log = 31;
    std::vector<u64> sizes(nf); std::vector<ZbSegment> out_segs(nf); u64 total = 0;
    simt::launch((nf + 255) / 256, 256, [&] { zb_frame_sizes(segs.data(), info.data(), outs.data(), nf, P, sizes.data()); });
    simt::launch(1, 1024, [&] { zb_scan_sizes(sizes.data(), nf, out_segs.data(), &total); });
    if (total > out_cap) return -1;
    simt::launch((nf + 7) / 8, 256, [&] { zb_write_frames(src, segs.data(), info.data(), outs.data(), slots.data(), slot_bytes, nf, P, out_segs.data(), out); });
    for (u32 f = 0; f < nf; f++) { out_off[f] = out_segs[f].offset; out_len[f] = out_segs[f].length; }
    return (long long)total;
}
"""


def build():
    """The encoder kernels' text exactly as host_encoder.build_compress_sim cuts it out of zb_encode.cu, with the chain driver."""
    os.makedirs(H.BUILD, exist_ok=True)
    csrc = os.path.join(H.ROOT, "python_zstandard_b200", "csrc")
    enc = open(H.SRC).read()
    a = enc.index("\n", enc.index('#include "zb_common.cuh"')) + 1
    b = enc.index('extern "C" {')
    b = enc.rindex("// ====", 0, enc.rindex("// ====", 0, b))
    body = enc[a:b].replace('#include "zb_encode2.cuh"', open(os.path.join(csrc, "zb_encode2.cuh")).read().replace("#pragma once", ""))
    body = body.replace('#include "zb_encode3.cuh"', open(os.path.join(csrc, "zb_encode3.cuh")).read().replace("#pragma once", ""))
    dec = open(os.path.join(csrc, "zb_decode.cu")).read()
    da = dec.index("\n", dec.index('#include "zb_common.cuh"')) + 1
    db = dec.index('extern "C" {')
    db = dec.rindex("// ====", 0, dec.rindex("// ====", 0, db))
    dbody = dec[da:db].replace('#include "zb_entropy.cuh"', open(H.DEC_SRC).read().replace("#pragma once", ""))
    body = re.sub(r"extern __shared__ __align__\(16\) u8 (\w+)\[\];", r"u8* const \1 = simt_dyn_smem;", dbody + body)
    text = (H.LIT_PRELUDE + "#include <cmath>\n#include <vector>\n" + '#include "%s"\n' % os.path.join(csrc, "zb_common.cuh")
            + '#include "%s"\n' % os.path.join(H.HERE, "simt.h") + "alignas(16) static u8 simt_dyn_smem[256 << 10];\n#define ZB_SIMT_STEP() __syncwarp()\n#define ZB_SIMT_EMULATION 1\n"
            + body + WRAPPERS)
    cpp = os.path.join(H.BUILD, "zc_chain_sim.cpp")
    if not (os.path.exists(LIB) and os.path.exists(cpp) and open(cpp).read() == text
            and os.path.getmtime(LIB) >= os.path.getmtime(os.path.join(H.HERE, "simt.h"))):
        open(cpp, "w").write(text)
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-o", LIB, cpp])
    L = C.CDLL(LIB)
    L.t_compress_chain_run.restype = C.c_longlong
    L.t_compress_chain_run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                       C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    return L


_batch = None


def first_frame(chunk, checksum=False, dict_data=None):
    """Chunk 0 through the CPU build of the batch path, content size on (dict_data: raw dictionary bytes or None)."""
    global _batch
    if _batch is None:
        _batch = H.build_compress_sim()
    data = np.frombuffer(bytes(chunk) + bytes(64), dtype=np.uint8)
    off, ln = np.array([0], np.uint64), np.array([len(chunk)], np.uint64)
    cap = len(chunk) + len(chunk) // 128 + 1024
    out = np.zeros(cap, np.uint8)
    o_off, o_len = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    d = bytes(dict_data) if dict_data else None
    n = _batch.t_compress_batch(data.ctypes.data, off.ctypes.data, ln.ctypes.data, 1, int(checksum), 1, 4, out.ctypes.data, cap,
                                o_off.ctypes.data, o_len.ctypes.data, 0, d, len(d) if d else 0, 3, 0)
    assert n > 0, n
    return out[int(o_off[0]):int(o_off[0] + o_len[0])].tobytes()


def one_run(k, sizes):
    return len(sizes)


def compress_chain(L, chunks, checksum=False, run_cut=one_run, dict_data=None, n_ctas=8):
    """Every frame of the chain, as zb200_compress_chain writes it.  run_cut(k, sizes) -> the end of the run whose first new
    chunk is k (the launcher's memory budget, made explicit); every run carries chunk k - 1 in as its prefix."""
    chunks = [bytes(c) for c in chunks]
    frames = [first_frame(chunks[0], checksum, dict_data)]
    sizes = [len(c) for c in chunks]
    k = 1
    while k < len(chunks):
        b = max(k + 1, min(run_cut(k, sizes), len(chunks)))
        run = chunks[k - 1:b]
        offs, pos = [], 64
        for c in run:
            offs.append(pos)
            pos += len(c)
        src = np.frombuffer(bytes(64) + b"".join(run) + bytes(64), dtype=np.uint8)
        offs = np.array(offs, np.uint64)
        lens = np.array([len(c) for c in run], np.uint64)
        nf = len(run) - 1
        cap = sum(len(c) + len(c) // 128 + 1024 for c in run[1:]) + 64
        out = np.zeros(cap, np.uint8)
        o_off, o_len = np.zeros(nf, np.uint64), np.zeros(nf, np.uint64)
        r = L.t_compress_chain_run(src.ctypes.data, offs.ctypes.data, lens.ctypes.data, len(run), int(checksum), n_ctas,
                                   out.ctypes.data, cap, o_off.ctypes.data, o_len.ctypes.data)
        assert r >= 0, r
        frames += [out[int(o):int(o + n)].tobytes() for o, n in zip(o_off, o_len)]
        k = b
    return frames
