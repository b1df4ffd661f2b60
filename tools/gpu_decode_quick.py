"""Quick device-resident decode timing (no CPU baselines, no compress arm) for kernel experiments."""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch, corpus
from oracle import RefZstd
import python_zstandard_b200 as zstd
from python_zstandard_b200 import _native
n = int(os.environ.get("N", "262144")); size = int(os.environ.get("SIZE", "4096"))
ref = RefZstd()
blob, off, ln = corpus.text_segments(n, size) if os.environ.get("MIX") is None else corpus.silesia_mix(n, size)
cblob, clens = ref.batch(True, blob, off, ln, level=3, threads=os.cpu_count())
coff = np.concatenate([[0], np.cumsum(clens)[:-1]]).astype(np.uint64)
segs = np.stack([coff, clens], axis=1).astype(np.uint64)
ctx = _native.Context.get(0); L = ctx.L
d_src = torch.empty(len(cblob) + 256, dtype=torch.uint8, device="cuda"); d_src[:len(cblob)].copy_(torch.from_numpy(cblob))
d_segs = torch.from_numpy(segs.view(np.int64).copy()).cuda()
def step():
    res = C.c_void_p()
    ctx.check(L.zb200_decompress_batch(ctx.h, d_src.data_ptr(), d_segs.data_ptr(), n, None, None, 3, C.byref(res)), "dec")
    return res
r = step()
out = np.empty(len(blob), dtype=np.uint8); L.zb200_memcpy_d2h(ctx.h, out.ctypes.data, L.zb200_result_data(r), len(blob)); L.zb200_result_free(r)
print("equal:", np.array_equal(out, blob))
for _ in range(3): L.zb200_result_free(step())
ctx.profile(True)
for _ in range(5): L.zb200_result_free(step())
p = ctx.profile_read()
tot = sum(v[0] / v[1] for v in p.values())
print({k: round(v[0] / v[1], 3) for k, v in p.items()}, "total ms %.3f -> %.1f GB/s" % (tot, len(blob) / tot / 1e6))
if os.environ.get("PHASES"):
    L.zb_entropy_phase_read.argtypes = [C.c_void_p, C.c_int]
    L.zb_execute_phase_read.argtypes = [C.c_void_p, C.c_int]
    buf = (C.c_uint64 * 8)(); L.zb_entropy_phase_read(buf, 1)
    xbuf = (C.c_uint64 * 4)(); L.zb_execute_phase_read(xbuf, 1)
    L.zb200_result_free(step()); L.zb_entropy_phase_read(buf, 1); L.zb_execute_phase_read(xbuf, 1)
    # slot 6 (Huffman claim + fill) and slot 7 (the three FSE builds) split phases B and D; a lane-0 mark, so when lane 0 has no
    # Huffman table or no sequences in a round, that round's table time stays with the streams or the sequence loop
    names = ['other/loop', 'A block header', 'B literals hdr+weights', 'huffman streams', 'C seq header+ncount', 'D sequence loop',
             'huffman table claim+fill', 'D FSE table builds']
    tot = float(sum(buf[i] for i in range(8))) or 1.0
    print('entropy phases (share of summed warp cycles):', {nm: "%.1f%% (%.0f Mcycles)" % (100.0 * buf[i] / tot, buf[i] / 1e6) for i, nm in enumerate(names)},
          "sum Mcycles %.0f" % (tot / 1e6))
    xnames = ['frame start + literal staging', 'literal copies', 'frontier passes', 'write-out']
    print('zb_execute_tile phases (summed warp cycles):', {nm: "%.1f Mcycles" % (xbuf[i] / 1e6) for i, nm in enumerate(xnames)},
          "sum Mcycles %.0f" % (sum(xbuf[i] for i in range(4)) / 1e6))
