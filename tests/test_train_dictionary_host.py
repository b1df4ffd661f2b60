"""The dictionary-training kernels (zb_train.cuh) on the CPU through tests/simt.h: frequency counts against a NumPy
restatement of FASTCOVER_computeFrequency, the previous-occurrence table against a direct scan, segment selection against
the reference's ZDICT_optimizeTrainFromBuffer_fastCover (equal dictionary IDs: the ID is XXH64 of every selected byte),
and finished dictionaries that the reference loads and uses."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

import corpus
from tests import train_ref

pytestmark = pytest.mark.skipif(not os.path.exists(train_ref.REF), reason="oracle/_ref is built from the reference sources")


@pytest.fixture(scope="module")
def sim():
    from tests import host_encoder
    return host_encoder.build_sim()


def foo_samples():
    inputs = [b"foo" * 64, b"bar" * 64, b"abcdef" * 64, b"sometext" * 64, b"baz" * 64]
    return [inputs[i % 5] for i in range(128)]


def corpora():
    text = corpus.text_corpus()[:120000].tobytes()    # (text_corpus caches its first length: ask for the default)
    rnd = np.random.default_rng(5).integers(0, 256, 60000).astype(np.uint8).tobytes()
    return {
        "json": corpus.json_records(200),
        "text": [text[i:i + 1500] for i in range(0, len(text), 1500)],
        "random": [rnd[i:i + 1000] for i in range(0, len(rnd), 1000)],
        "foo": foo_samples(),
    }


def layout(samples, split):
    n = len(samples)
    n_train = int(n * split) if split < 1.0 else n
    blob = b"".join(samples) + bytes(16)
    offs = np.cumsum([0] + [len(s) for s in samples]).astype(np.uint64)
    return blob, offs, n_train


def np_hash(blob, pos, f, d):
    b = np.frombuffer(blob, dtype=np.uint8)
    v = np.zeros(len(pos), dtype=np.uint64)
    for i in range(7, -1, -1):
        v = (v << np.uint64(8)) | b[pos + i].astype(np.uint64)
    with np.errstate(over="ignore"):
        if d == 6:
            h = ((v << np.uint64(16)) * np.uint64(227718039650203)) >> np.uint64(64 - f)
        else:
            h = (v * np.uint64(0xCF1BBCDCB7A56463)) >> np.uint64(64 - f)
    return h


def np_freqs(blob, offs, n_train, f, d, step):
    """FASTCOVER_computeFrequency (zstd/zstd.c:52074): training samples, every step-th position while 8 bytes remain."""
    pos = [np.arange(int(offs[i]), int(offs[i + 1]) - 7, step, dtype=np.int64) for i in range(n_train)]
    pos = np.concatenate(pos) if pos else np.zeros(0, np.int64)
    return np.bincount(np_hash(blob, pos, f, d).astype(np.int64), minlength=1 << f).astype(np.uint32)


@pytest.mark.parametrize("d,f,accel,split", list(itertools.product((6, 8), (10, 16, 20), (1, 2, 10), (1.0, 0.75))))
def test_counts_equal_a_numpy_restatement(sim, d, f, accel, split):
    recs = corpus.json_records(60)
    samples = recs[:20] + [b"", b"a", b"abcdefg", b"12345678", b"123456789"] + recs[20:]     # shorter than 8 bytes too
    blob, offs, n_train = layout(samples, split)
    out = np.zeros(1 << f, dtype=np.uint32)
    sim.t_freqs(blob, offs.ctypes.data, n_train, f, d, accel, out.ctypes.data)
    assert np.array_equal(out, np_freqs(blob, offs, n_train, f, d, accel))


def test_previous_occurrence_table(sim):
    """prev[j]: the last position before j with the same hash, across the 4096-position chunks of the sort."""
    rng = np.random.default_rng(3)
    n = 3 * 4096 + 77
    h = rng.integers(0, 300, n).astype(np.uint32)
    prev = np.zeros(n, dtype=np.uint32)
    sim.t_prev(h.ctypes.data, n, 9, prev.ctypes.data)
    last = {}
    want = np.empty(n, dtype=np.uint32)
    for j, x in enumerate(h.tolist()):
        want[j] = last.get(x, 0xFFFFFFFF)
        last[x] = j
    assert np.array_equal(prev, want)


def our_content(sim, samples, k, d, f, accel, split, cap):
    blob, offs, n_train = layout(samples, split)
    dct = (C.c_ubyte * cap)()
    tail = C.c_uint32(0)
    sim.t_select(blob, offs.ctypes.data, n_train, f, d, accel, k, cap, dct, C.byref(tail))
    return bytes(dct)[tail.value:]


def compliant_id(content):
    from oracle import Oracle
    return Oracle().xxh64(content) % ((1 << 31) - 32768) + 32768


GRID = [(k, d, f, accel, split, cap) for (k, d, split), (f, accel, cap) in
        zip(itertools.product((50, 64, 500, 1998), (6, 8), (0.75, 1.0)),
            itertools.cycle(itertools.product((16, 20), (1, 4), (256, 8192, 112640))))]


@pytest.mark.parametrize("name", ["json", "text", "random", "foo"])
def test_selection_equals_the_reference(sim, name):
    samples = corpora()[name]
    for k, d, f, accel, split, cap in GRID:
        if k > cap:
            continue
        try:
            ref, _, _ = train_ref.train_fastcover(cap, samples, k=k, d=d, f=f, accel=accel, split_point=split, steps=1)
        except train_ref.TrainError:
            continue                 # the reference's finalisation refused this corpus / capacity: nothing to compare
        content = our_content(sim, samples, k, d, f, accel, split, cap)
        assert compliant_id(content) == train_ref.dict_id(ref), (name, k, d, f, accel, split, cap)


def test_epoch_wrap_and_clamp(sim):
    """A corpus whose epoch size is clamped to 10 k (few d-mers per epoch) and whose visits wrap around the epochs
    several times before the capacity is full."""
    samples = corpus.json_records(40)
    for k, d, cap in ((200, 8, 112640), (1998, 6, 8192), (50, 6, 112640)):
        ref, _, _ = train_ref.train_fastcover(cap, samples, k=k, d=d, split_point=1.0, steps=1)
        content = our_content(sim, samples, k, d, 20, 1, 1.0, cap)
        assert compliant_id(content) == train_ref.dict_id(ref), (k, d, cap)


def test_finished_dictionary_loads_in_the_reference(sim):
    """zt_entropy + zt_finalize: the reference codec loads the dictionary (header, Huffman table, NCounts, repcodes) and
    round-trips records with it; a dict_id given is written as is."""
    from oracle import RefZstd
    ref = RefZstd()
    recs = corpus.json_records(300)
    content = our_content(sim, recs[:200], 500, 8, 20, 1, 1.0, 16384)[-8000:]     # room for the header: nothing shrinks
    cap = 16384
    dct = (C.c_ubyte * cap).from_buffer_copy(bytes(cap - len(content)) + content)
    rng = np.random.default_rng(9)
    stats = np.zeros(512, dtype=np.uint32)
    stats[:256] = rng.integers(0, 5000, 256)
    stats[256:292] = rng.integers(0, 900, 36)
    stats[292:345] = rng.integers(0, 900, 53)
    stats[345:363] = rng.integers(0, 900, 18)
    out = (C.c_ubyte * cap)()
    for dict_id in (0, 42):
        n = sim.t_finalize(dct, cap, cap - len(content), stats.ctypes.data, dict_id, out)
        assert n > 0
        d = bytes(out)[:n]
        assert d[:4] == b"\x37\xa4\x30\xec" and d.endswith(content)
        assert train_ref.dict_id(d) == (dict_id or compliant_id(content))
        for r in recs[200:230]:
            assert ref.decompress(ref.compress(r, level=3, dict_data=d), len(r), d) == r
