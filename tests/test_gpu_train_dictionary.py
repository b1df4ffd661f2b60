"""train_dictionary on the device: the reference's scenarios (tests/test_train_dictionary.py of python-zstandard), exact
segment selection against the reference's fastCover (equal dictionary IDs: the ID hashes every selected byte), the
error texts, and round trips / sizes with the trained dictionaries."""
import os

import pytest

import corpus
import python_zstandard_b200 as zstd
from tests import train_ref

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.exists(train_ref.REF), reason="oracle/_ref is built from the reference sources")]


def generate_samples():
    """The reference test's samples: runs that leave most epochs without a new d-mer (zero-score visits)."""
    inputs = [b"foo" * 64, b"bar" * 64, b"abcdef" * 64, b"sometext" * 64, b"baz" * 64]
    return [inputs[i % 5] for i in range(128)]


def test_no_args():
    with pytest.raises(TypeError):
        zstd.train_dictionary()


def test_bad_args():
    with pytest.raises(TypeError):
        zstd.train_dictionary(8192, "foo")
    with pytest.raises(ValueError):
        zstd.train_dictionary(8192, ["foo"])


def test_no_params():
    d = zstd.train_dictionary(8192, generate_samples())
    assert isinstance(d.dict_id(), int)
    data = d.as_bytes()
    assert data[0:4] == b"\x37\xa4\x30\xec"
    assert d.k == 50 and d.d == 8


def test_basic():
    d = zstd.train_dictionary(8192, generate_samples(), k=500, d=8)
    assert d.k == 500 and d.d == 8
    assert d.dict_id() == train_ref.dict_id(train_ref.train_fastcover(8192, generate_samples(), k=500, d=8)[0])


def test_set_dict_id():
    d = zstd.train_dictionary(8192, generate_samples(), k=64, d=8, dict_id=42)
    assert d.dict_id() == 42


def test_optimize():
    d = zstd.train_dictionary(8192, generate_samples(), threads=-1, steps=1, d=6)
    assert d.k in (50, 2000)
    assert d.d == 6


def _corpora():
    recs = corpus.json_records(3000)
    text = corpus.text_corpus()[:300000].tobytes()    # (text_corpus caches its first length: ask for the default)
    import numpy as np
    rnd = np.random.default_rng(5).integers(0, 256, 200000).astype(np.uint8).tobytes()
    return {
        "json": recs[:2000],
        "text": [text[i:i + 1500] for i in range(0, len(text), 1500)],
        "random": [rnd[i:i + 1000] for i in range(0, len(rnd), 1000)],
        "foo": generate_samples(),
        "tiny": recs[:40] + [b"ab", b"", b"xyz1234"],                      # smaller than most capacities: tail left over
    }


@pytest.mark.parametrize("name", ["json", "text", "random", "foo", "tiny"])
def test_selection_matches_the_reference(name):
    """For a fixed (k, d) the content is the reference's: equal IDs (XXH64 of the whole pre-shrink content)."""
    samples = _corpora()[name]
    grid = [(50, 8, 20, 1, 0.75, 8192), (64, 6, 16, 4, 1.0, 8192), (500, 8, 16, 1, 1.0, 112640), (1998, 6, 20, 4, 0.75, 112640),
            (50, 6, 20, 1, 1.0, 256), (200, 8, 20, 4, 0.75, 256)]
    for k, d, f, accel, split, cap in grid:
        try:
            ref, rk, rd = train_ref.train_fastcover(cap, samples, k=k, d=d, f=f, accel=accel, split_point=split, steps=1)
        except train_ref.TrainError as e:      # the reference refuses this corpus / capacity: so must we, with its words
            with pytest.raises(zstd.ZstdError, match="cannot train dict: " + str(e)):
                zstd.train_dictionary(cap, samples, k=k, d=d, f=f, accel=accel, split_point=split, steps=1)
            continue
        ours = zstd.train_dictionary(cap, samples, k=k, d=d, f=f, accel=accel, split_point=split, steps=1)
        assert (ours.k, ours.d) == (rk, rd) == (k, d)
        assert ours.dict_id() == train_ref.dict_id(ref), (name, k, d, f, accel, split, cap)
        assert len(ours) <= cap
        if len(ref) < cap and len(ours) < cap:                 # nothing shrunk: the contents are the same bytes
            m = min(len(ref), len(ours)) - 300
            assert m <= 0 or ours.as_bytes()[-m:] == ref[-m:]


@pytest.mark.parametrize("kwargs,margin", [(dict(k=1024, d=8), 1.01), (dict(), 1.02), (dict(threads=-1), 1.02)])
def test_bench_call_sizes_and_round_trips(kwargs, margin):
    """train_dictionary(112640, recs[:2000]) as the dictionary benchmark calls it, with an explicit (k, d), with the
    defaults and with the 82-candidate search.  16384 held-out records compressed by this package with our dictionary and
    with the reference's: with (k, d) given the contents are the same and only the entropy tables differ (within 1 %);
    under the search the chosen k may differ, since candidates are scored with this package's compressor (within 2 %)."""
    from oracle import RefZstd
    ref = RefZstd()
    recs = corpus.json_records(2000 + 16384)
    train, held = recs[:2000], recs[2000:]
    ours = zstd.train_dictionary(112640, train, **kwargs)
    theirs_b, tk, td = train_ref.train_fastcover(112640, train, **kwargs)
    theirs = zstd.ZstdCompressionDict(theirs_b)
    sizes = {}
    for tag, dct in (("ours", ours), ("ref", theirs)):
        out = zstd.ZstdCompressor(level=3, dict_data=dct).multi_compress_to_buffer(held)
        sizes[tag] = sum(len(out[i]) for i in range(len(held)))
        back = zstd.ZstdDecompressor(dict_data=dct).multi_decompress_to_buffer(out)
        assert all(back[i].tobytes() == held[i] for i in range(len(held)))
        for i in range(0, len(held), 997):
            assert ref.decompress(out[i].tobytes(), len(held[i]), dct.as_bytes()) == held[i]
    sizes["ref_codec_ours"] = sum(len(ref.compress(r, level=3, dict_data=ours.as_bytes())) for r in held[:2048])
    sizes["ref_codec_ref"] = sum(len(ref.compress(r, level=3, dict_data=theirs_b)) for r in held[:2048])
    print("train_dictionary %s: k=%d d=%d (reference k=%d d=%d), held-out sizes %s" % (kwargs, ours.k, ours.d, tk, td, sizes))
    if "k" in kwargs:
        assert ours.dict_id() == train_ref.dict_id(theirs_b)
    assert sizes["ours"] <= sizes["ref"] * margin, sizes


@pytest.mark.parametrize("args", [
    dict(dict_size=8192, samples=corpus.json_records(4)),
    dict(dict_size=255, samples=generate_samples()),
    dict(dict_size=8192, samples=generate_samples(), d=7),
    dict(dict_size=8192, samples=generate_samples(), k=4, d=6),
    dict(dict_size=8192, samples=generate_samples(), accel=11),
    dict(dict_size=8192, samples=generate_samples(), f=32, k=100, d=8),
    dict(dict_size=8192, samples=generate_samples(), split_point=1.5),
])
def test_error_texts(args):
    """The reference's ZDICT error for the same arguments, under the reference's message."""
    with pytest.raises(train_ref.TrainError) as ref_err:
        train_ref.train_fastcover(**args)
    with pytest.raises(zstd.ZstdError) as our_err:
        zstd.train_dictionary(**args)
    assert str(our_err.value) == "cannot train dict: " + str(ref_err.value)
