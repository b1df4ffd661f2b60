"""The chain encoder (compress_content_dict_chain) on the CPU: the launchers of zb_chain_index, the prefix mode of
zb_compress_blocks and the frame layout kernels on tests/simt.h (t_compress_chain_run of host_encoder.build_sim), driven run
by run as zb200_compress_chain (zb_api.cu) drives them on the device.  Chunk 0 goes through the CPU build of the batch path
(t_compress_batch), as the launcher sends it through zb200_compress_batch_ptrs.
TEST INFRASTRUCTURE, NOT PRODUCT CODE."""
import ctypes as C

import numpy as np

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


def first_frame(L, chunk, checksum=False, dict_data=None):
    """Chunk 0 through the CPU build of the batch path, content size on (dict_data: raw dictionary bytes or None)."""
    data = np.frombuffer(bytes(chunk) + bytes(64), dtype=np.uint8)
    off, ln = np.array([0], np.uint64), np.array([len(chunk)], np.uint64)
    cap = len(chunk) + len(chunk) // 128 + 1024
    out = np.zeros(cap, np.uint8)
    o_off, o_len = np.zeros(1, np.uint64), np.zeros(1, np.uint64)
    d = bytes(dict_data) if dict_data else None
    n = L.t_compress_batch(data.ctypes.data, off.ctypes.data, ln.ctypes.data, 1, int(checksum), 1, 4, out.ctypes.data, cap,
                                o_off.ctypes.data, o_len.ctypes.data, 0, d, len(d) if d else 0, 3, 0)
    assert n > 0, n
    return out[int(o_off[0]):int(o_off[0] + o_len[0])].tobytes()


def one_run(k, sizes):
    return len(sizes)


def compress_chain(L, chunks, checksum=False, run_cut=one_run, dict_data=None, n_ctas=8):
    """Every frame of the chain, as zb200_compress_chain writes it.  run_cut(k, sizes) -> the end of the run whose first new
    chunk is k (the launcher's memory budget, made explicit); every run carries chunk k - 1 in as its prefix."""
    chunks = [bytes(c) for c in chunks]
    frames = [first_frame(L, chunks[0], checksum, dict_data)]
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
