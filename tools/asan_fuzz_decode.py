"""AddressSanitizer fuzz of the decode kernels' source on the CPU (t_decode_frame of tests/host_encoder.build_sim: one
frame through the launchers and the lane-per-frame entropy kernel): mutated and truncated golden frames in exact-size heap
blocks with PAD bytes of slack on both sides.
  ASAN_OPTIONS=detect_leaks=0 LD_PRELOAD=$(gcc -print-file-name=libasan.so) N=50 SEED=1 python tools/asan_fuzz_decode.py
The default PAD=16 covers the bit reader's by-design reads: it copies the 16-byte aligned chunks that cover a stream (up to 15
bytes past the segment, inside its allocation granule on the device); smaller PADs show those reads.
The kernels run on simt.h's ucontext fibers, which ASan supports only in part (it warns about makecontext / swapcontext):
check a report against the fiber stacks first.  N=50 SEED=1: 800 fuzzed, 230 accepted, no report (~8 minutes once
built)."""
import sys, os, ctypes as C, numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import helpers, host_encoder
L=host_encoder.build_sim("/tmp/libzsim_asan.so", ["-O1", "-g", "-fsanitize=address", "-fno-omit-frame-pointer"])
PAD=int(os.environ.get('PAD','16'))
libc=C.CDLL(None); libc.malloc.restype=C.c_void_p; libc.malloc.argtypes=[C.c_size_t]; libc.free.argtypes=[C.c_void_p]
def decode(frame,cap,dct=b''):
    # exact-size heap blocks so that ASAN red zones sit right behind the data (+PAD slack on both sides)
    n=len(frame); sp=libc.malloc(n+2*PAD); C.memset(sp,0,n+2*PAD); C.memmove(sp+PAD,frame,n)
    dp=None
    if dct:
        dp=libc.malloc(len(dct)+2*PAD); C.memset(dp,0,len(dct)+2*PAD); C.memmove(dp+PAD,dct,len(dct))
    op=libc.malloc(cap+2*PAD if cap+2*PAD else 1)
    on,nb,ns=C.c_uint64(0),C.c_uint32(0),C.c_uint32(0)
    rc=L.t_decode_frame(sp+PAD,n,(dp+PAD) if dct else None,len(dct),op+PAD,cap,C.byref(on),C.byref(nb),C.byref(ns))
    libc.free(sp); libc.free(op)
    if dp: libc.free(dp)
    return rc
rng=np.random.default_rng(int(os.environ.get('SEED','1')))
vecs=helpers.golden_vectors()
tot=acc=0
for name,frame,raw,dct in vecs:
    assert decode(frame,len(raw),dct)==0,name
    for t in range(int(os.environ.get('N','300'))):
        bad=bytearray(frame)
        for _ in range(int(rng.integers(1,4))):
            k=int(rng.integers(0,len(bad))); bad[k]=int(rng.integers(0,256)) if t%2 else bad[k]^(1<<int(rng.integers(0,8)))
        if t%7==0: bad=bad[:int(rng.integers(1,len(bad)+1))]
        rc=decode(bytes(bad),len(raw),dct); tot+=1; acc+=rc==0
print('fuzzed',tot,'accepted',acc)
