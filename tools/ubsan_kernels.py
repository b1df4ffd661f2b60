"""UndefinedBehaviorSanitizer over the CPU builds of ALL kernels (tests/simt.h): compress (default, two-table, dictionary)
and the whole decode pipeline on KATs, text, 128 KiB blocks, zeros, noise, dictionary records and reference-made frames.
   python tools/ubsan_kernels.py          (round 1: no report -- no out-of-range shift, signed overflow or misaligned access)"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import host_encoder
Lc=Ld=host_encoder.build_sim("/tmp/libzsim_ubsan.so",["-O1","-g","-fsanitize=undefined"])
print("built")
import tests.test_compress_kernel_host as tc, tests.test_decode_pipeline_host as td
from oracle import RefZstd
import corpus, numpy as np
ref=RefZstd()
text=corpus.text_corpus(1<<20)
segs=[b"foo"*12,b"",bytes(text[:4096]),bytes(text[5000:6500]),bytes(text[10000:10000+131072]),bytes(9000),np.random.default_rng(1).integers(0,256,7000).astype(np.uint8).tobytes()]
for dual in (False,True):
    fr=tc.compress(Lc,segs,checksum=True,n_ctas=2,dual=dual)
    outs,st=td.decompress(Ld,fr,[len(s) for s in segs],n_ctas=1)
    print("dual",dual,st,outs==segs)
recs=corpus.json_records(440); dct=ref.train_dictionary(16384,recs[:400])
fr=tc.compress(Lc,recs[400:],n_ctas=2,dct=dct)
outs,st=td.decompress(Ld,fr,[len(r) for r in recs[400:]],dct)
print("dict",set(st),outs==recs[400:])
frames=[ref.compress(s,level=l,checksum=True) for s,l in zip(segs,(3,3,1,5,19,3,3))]
outs,st=td.decompress(Ld,frames,[len(s) for s in segs],n_ctas=1,warps=7,take=16)
print("ref frames",st,outs==segs)
