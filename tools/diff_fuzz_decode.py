"""Differential fuzz on the CPU: the decode kernels' source (t_decode_frame of tests/host_encoder.build_sim: one frame through
the launchers and the lane-per-frame entropy kernel) against the unmodified reference on mutated frames (text at several
levels, Silesia-mix members, dictionary records; no content checksum so that the reference accepts many mutations).
   N=300 SEED=5 python tools/diff_fuzz_decode.py
A frame costs ~0.1 s, nearly all of it the placement's two CTAs of 1024 fibers: N=300 (8100 frames) takes ~13 minutes, the
default N=2000 (54000 frames) about 1.5 hours.  N=300 SEED=5: 3222 both accept with equal bytes, 4218 both reject, 660 the
kernel code rejects alone (the exact-consumption rule of the literal streams), 0 accepted against the reference, 0 byte
mismatches."""
import sys, os, ctypes as C, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import helpers, host_encoder
from tests.test_entropy_kernel_host import decode
from oracle import RefZstd, Oracle
import corpus
kern=host_encoder.build_sim(); ref=RefZstd(); orc=Oracle()
rng=np.random.default_rng(int(os.environ.get('SEED','5')))
blob=corpus.text_corpus(1<<20)
frames=[]
for size,level in ((200,3),(1500,3),(4096,3),(4096,1),(4096,-1),(20000,5),(70000,3),(140000,3),(9000,19)):
    o=int(rng.integers(0,len(blob)-size)); data=bytes(blob[o:o+size]); frames.append((ref.compress(data,level=level,checksum=False),data,b''))
mix,off,ln=corpus.silesia_mix(8,30000)
for o,l in zip(off,ln):
    d=bytes(mix[int(o):int(o)+int(l)]); frames.append((ref.compress(d,level=3,checksum=False),d,b''))
recs=corpus.json_records(500); dct=ref.train_dictionary(16384,recs[:400])
for r in recs[400:410]: frames.append((ref.compress(r,level=3,dict_data=dct,checksum=False),r,dct))
N=int(os.environ.get('N','2000'))
both=rej=strict=bad_accept=mismatch=0
for frame,data,d in frames:
    for t in range(N):
        b=bytearray(frame)
        for _ in range(1 if t%3 else 2):
            k=int(rng.integers(4,len(b)))
            if t%2: b[k]^=1<<int(rng.integers(0,8))
            else: b[k]=int(rng.integers(0,256))
        try: want=ref.decompress(bytes(b),len(data),d)
        except RefZstd.Error: want=None
        rc,got,_,_=decode(kern,bytes(b),len(data),d)
        if want is None:
            if rc==0:
                bad_accept+=1
                if bad_accept<=5: print('ACCEPTED what the reference rejects: frame len',len(frame),'mut',bytes(b).hex()[:80])
            else: rej+=1
        elif rc==0:
            if got!=want:
                mismatch+=1
                if mismatch<=5: print('MISMATCH len',len(frame))
            else: both+=1
        else: strict+=1
print('both accept & equal',both,'both reject',rej,'kernel stricter',strict,'BAD accept',bad_accept,'MISMATCH',mismatch)
