"""Encoder fuzz (dev container: needs oracle/_ref): kernel source on the host / emulated warp vs the compiled reference on generated inputs of many shapes, levels and frame flags.  usage: python scripts/fuzz_encoder_vs_ref.py <seed> <seconds> [emu]
Levels 13..22 (optimal parser) run on the first 64 KB of the input, through tests/hostsim/libzb_hostsim_opt.so."""
import sys, random, time
sys.path.insert(0, __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__))))
import numpy as np
from tests.oracle_util import *
from tests.test_opt_levels import host as opt_compress
seed=int(sys.argv[1]); T=float(sys.argv[2]); emu=len(sys.argv)>3
rnd=random.Random(seed); rng=np.random.default_rng(seed)
def gen():
    n=rnd.choice([rnd.randint(0,300), rnd.randint(300,20000), rnd.randint(16000,17000), rnd.randint(20000,131072), 131072, 131072])
    kind=rnd.randrange(8)
    if kind==0: a=rng.integers(0,rnd.choice([2,4,16,64,256]),n,dtype=np.uint8)
    elif kind==1:
        motif=rng.integers(0,256,rnd.randint(1,5000),dtype=np.uint8); a=np.resize(motif,n).copy()
        m=rng.random(n)<rnd.choice([0,0.001,0.01,0.1]); a[m]=rng.integers(0,256,int(m.sum()),dtype=np.uint8)
    elif kind==2:
        a=np.cumsum(rng.integers(-3,4,n)).astype(np.uint8)
    elif kind==3:
        words=[bytes(rng.integers(97,123,rnd.randint(2,9),dtype=np.uint8)) for _ in range(rnd.randint(5,400))]
        s=b" ".join(rnd.choice(words) for _ in range(n//4+1))[:n]; a=np.frombuffer(s,dtype=np.uint8)
    elif kind==4:
        a=np.zeros(n,dtype=np.uint8); k=rnd.randint(0,20)
        for _ in range(k):
            if n: a[rnd.randrange(n)]=rnd.randrange(256)
    elif kind==5:
        rec=rng.integers(0,256,64,dtype=np.uint8); a=np.tile(rec,n//64+1)[:n].copy(); idx=np.arange(n)%64>=rnd.randint(16,60); a[idx]=rng.integers(0,256,int(idx.sum()),dtype=np.uint8)
    elif kind==6:
        p=rng.dirichlet(np.ones(256)*rnd.choice([0.05,0.3,1.0])); a=rng.choice(256,n,p=p).astype(np.uint8)
    else:
        parts=[]; left=n
        while left>0:
            k=min(left,rnd.randint(1,30000)); t=rnd.randrange(3)
            parts.append(rng.integers(0,256,k,dtype=np.uint8) if t==0 else np.full(k,rnd.randrange(256),dtype=np.uint8) if t==1 else np.resize(rng.integers(0,50,rnd.randint(1,300),dtype=np.uint8),k)); left-=k
        a=np.concatenate(parts) if parts else np.zeros(0,dtype=np.uint8)
    return a.tobytes()
t0=time.time(); n=0; bad=0
while time.time()-t0<T:
    d=gen(); lvl=rnd.choice([1,2,3,3,3,4,5,6,7,8,9,10,11,12,-1,-5,-50]+list(range(13,23)))
    if lvl>=13: d=d[:65536]
    if len(d)<=16384 and lvl in (11,12): continue
    ck=rnd.random()<0.2; cs=rnd.random()<0.8
    e=ref_compress_flags(d,lvl,ck,cs,False)
    if lvl>=13: g=opt_compress(d,lvl,flags={"checksum":ck,"content_size":cs},emu=emu and rnd.random()<0.3)
    elif emu and lvl in (1,2,3,4,-1,-5,-50,5,6,7,8,9,10) and not ck and cs: g=emu_compress(d,lvl)
    else: g=hostsim_compress_flags(d,lvl,ck,cs)
    n+=1
    if e!=g:
        bad+=1; print("MISMATCH",seed,n,len(d),lvl,ck,cs,e if isinstance(e,int) else len(e), g if isinstance(g,int) else len(g)); open(f"/tmp/fuzz_enc_bad_{seed}_{n}.bin","wb").write(d)
print("seed",seed,"cases",n,"bad",bad)
