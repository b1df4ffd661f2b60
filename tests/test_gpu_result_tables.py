"""Segment tables of batch-decode results.  A device-resident result (ZB200_DST_DEVICE) keeps its table on the device, in
its own allocation, until zb200_result_segments first asks for it; the host tables are blocks of the context's pinned
pool, and zb200_result_free hands them back."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

import corpus
from oracle import RefZstd, have_ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not have_ref(), reason="needs the reference codec built into oracle/_ref")]


def _batch(seed, n):
    rng = np.random.default_rng(seed)
    text = corpus.text_corpus(1 << 20)
    items = [text[o:o + int(s)].tobytes() for o, s in zip(rng.integers(0, (1 << 20) - 20000, n), rng.integers(0, 20000, n))]
    ref = RefZstd()
    frames = [ref.compress(s, level=3) for s in items]
    lens = np.array([len(f) for f in frames], dtype=np.uint64)
    segs = np.stack([np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64), lens], axis=1).astype(np.uint64)
    return items, np.frombuffer(b"".join(frames), dtype=np.uint8).copy(), segs


def _table(L, r):
    n = L.zb200_result_count(r)
    p = L.zb200_result_segments(r)
    assert p
    return p, np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint64)), shape=(n, 2)).copy()


class _Calls:
    def __init__(self, blob, segs):
        from python_zstandard_b200 import _native
        self.L, self.ctx, self.N = _native.lib(), _native.Context.get(0), _native
        self.blob, self.segs, self.n = blob, segs, len(segs)
        self.d_src = torch.from_numpy(blob).cuda()
        self.d_segs = torch.from_numpy(segs.view(np.int64).copy()).cuda()
        torch.cuda.synchronize()

    def device(self):
        r = C.c_void_p()
        self.ctx.check(self.L.zb200_decompress_batch(self.ctx.h, self.d_src.data_ptr(), self.d_segs.data_ptr(), self.n, None, None,
                                                     self.N.SRC_DEVICE | self.N.DST_DEVICE, C.byref(r)), "zb200_decompress_batch")
        return r

    def host(self):
        r = C.c_void_p()
        self.ctx.check(self.L.zb200_decompress_batch(self.ctx.h, self.blob.ctypes.data, self.segs.ctypes.data, self.n, None, None,
                                                     0, C.byref(r)), "zb200_decompress_batch")
        return r

    def device_items(self, r, table):
        size = int(self.L.zb200_result_size(r))
        out = np.empty(size, dtype=np.uint8)
        self.ctx.check(self.L.zb200_memcpy_d2h(self.ctx.h, out.ctypes.data, self.L.zb200_result_data(r), size), "d2h")
        return [out[int(o):int(o) + int(n)].tobytes() for o, n in table]


def test_a_lazy_table_read_after_the_next_call_is_the_first_calls():
    items_a, blob_a, segs_a = _batch(1, 700)
    items_b, blob_b, segs_b = _batch(2, 300)
    a, b = _Calls(blob_a, segs_a), _Calls(blob_b, segs_b)
    L = a.L
    ra = a.device()
    rb = b.device()                                  # a second call on the same context before ra's table is read
    rb2 = b.device()
    _, ta = _table(L, ra)
    assert [int(n) for _, n in ta] == [len(s) for s in items_a]
    assert a.device_items(ra, ta) == items_a
    # the same table as the host path's, which copies it into pinned memory inside the call
    rh = a.host()
    _, th = _table(L, rh)
    assert np.array_equal(ta, th)
    base = L.zb200_result_data(rh)
    assert [C.string_at(base + int(o), int(n)) for o, n in th] == items_a
    p1, again = _table(L, ra)
    assert p1 == L.zb200_result_segments(ra) and np.array_equal(again, ta)      # read once, the same array after
    _, tb = _table(L, rb2)
    assert b.device_items(rb2, tb) == items_b
    for r in (ra, rb, rb2, rh):
        assert not L.zb200_result_first_error(r, None, None, None, None)
        L.zb200_result_free(r)


def test_freed_results_give_their_pinned_tables_back():
    """A result's pinned table returns to the context's pool on zb200_result_free: the next result of the same size gets the
    same block, however many calls follow (a block still marked busy would make the pool allocate a new one)."""
    gc.collect()
    items, blob, segs = _batch(3, 500)
    calls = _Calls(blob, segs)
    L = calls.L
    blocks = []
    for make in (calls.device, calls.host):
        r = make()
        first, t0 = _table(L, r)
        blocks.append(first)
        L.zb200_result_free(r)
        for _ in range(4):
            r = make()
            p, t = _table(L, r)
            assert p == first and np.array_equal(t, t0)
            L.zb200_result_free(r)
    # results never read do not take a block: the next read still finds the same one free.  Their device memory (output
    # and table) goes back to the stream-ordered pool, which keeps it: the device's free memory does not shrink per call
    L.zb200_result_free(calls.device())
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(6):
        L.zb200_result_free(calls.device())
    assert free0 - torch.cuda.mem_get_info()[0] < sum(len(s) for s in items)
    r = calls.device()
    p, t = _table(L, r)
    assert p == blocks[0] and calls.device_items(r, t) == items
    L.zb200_result_free(r)
