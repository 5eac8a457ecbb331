"""Differential test of the JPEG coefficient codec (csrc/jpegcoef.c) on random files: Pillow writes JPEGs of
random size / quality / sub-sampling / Huffman optimisation / restart intervals / progressive mode, and the
lossless transcode (`jpegqs -n 0`) must give the same bytes with the one-thread reader, with the threaded
reader (random thread count and chunk size) and with the reference's own quantsmooth.c on libjpeg-turbo
(oracle/_ref/refcli_cpu, built by oracle/Makefile).  Without refcli_cpu the SHA-256 of its files stored for
this seed in tests/golden/reference/ref_files.json stand in for it; --record prints them (as the last line, JSON).
No GPU needed.
    python tools/codec_difftest.py [seed] [files] [--record]   (in a scratch directory: it writes in.jpg, s.jpg, p.jpg, r.jpg)"""
import hashlib, json, os, subprocess, sys, numpy as np
from PIL import Image
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E=os.path.join(ROOT,"jpeg-quantsmooth_b200","csrc","jpegqs"); R=os.path.join(ROOT,"oracle","_ref","refcli_cpu")
record="--record" in sys.argv; argv=[a for a in sys.argv[1:] if a!="--record"]
seed=int(argv[0]) if argv else 1
rng=np.random.RandomState(seed)
N=int(argv[1]) if len(argv)>1 else 200
want=None
if not os.path.exists(R):
    assert not record, "--record needs oracle/_ref/refcli_cpu"
    with open(os.path.join(ROOT,"tests","golden","reference","ref_files.json")) as f: want=json.load(f)["codec_difftest"][str(seed)]
    assert len(want)>=N, f"only {len(want)} files stored for seed {seed}"
sha=lambda b: hashlib.sha256(b).hexdigest()
digests=[]
bad=0
for it in range(N):
    w=int(rng.randint(8,900)); h=int(rng.randint(8,700)); gray=rng.rand()<0.2
    kind=rng.randint(4)
    y,x=np.mgrid[0:h,0:w]
    base=128+rng.randint(10,90)*np.sin(x/rng.uniform(3,80))+rng.randint(10,60)*np.cos(y/rng.uniform(3,80))
    noise=rng.normal(0,rng.choice([0.5,3,10,40]),(h,w,3))
    img=(np.stack([base,base[::-1],base[:,::-1]],-1)+noise).clip(0,255).astype(np.uint8)
    im=Image.fromarray(img,"RGB")
    if gray: im=im.convert("L")
    kw=dict(quality=int(rng.choice([1,5,20,50,75,90,95,100])))
    if not gray: kw["subsampling"]=int(rng.randint(3))
    if rng.rand()<0.3: kw["optimize"]=True
    r=rng.rand()
    if r<0.25: kw["restart_marker_rows"]=int(rng.randint(1,5))
    elif r<0.5: kw["restart_marker_blocks"]=int(rng.randint(1,40))
    if rng.rand()<0.15: kw["progressive"]=True
    try:
        im.save("in.jpg",**kw)
    except OSError:
        digests.append(None); continue
    env=dict(os.environ,JPEGQS_SERIAL_DECODE="1",JPEGQS_CODEC_THREADS="1")
    assert subprocess.run([E,"-n","0","-i","0","in.jpg","s.jpg"],env=env).returncode==0,(it,kw)
    th=str(int(rng.randint(4,17))); mb=str(int(rng.choice([64,300,2000,20000])))
    env=dict(os.environ,JPEGQS_CODEC_THREADS=th,JPEGQS_PAR_MIN_BYTES=mb,JPEGQS_CODEC_TRACE="1")
    p=subprocess.run([E,"-n","0","-i","0","in.jpg","p.jpg"],env=env,capture_output=True,text=True)
    assert p.returncode==0,(it,kw,p.stderr)
    a,b=(open(f,"rb").read() for f in ("s.jpg","p.jpg"))
    if want is None:
        assert subprocess.run([R,"-n","0","-i","0","in.jpg","r.jpg"]).returncode==0
        c=sha(open("r.jpg","rb").read())
    else:
        c=want[it]
    digests.append(c)
    if not (a==b and sha(a)==c):
        bad+=1; print("MISMATCH",it,w,h,gray,kw,th,mb,a==b,a==c); os.rename("in.jpg",f"bad{it}.jpg")
    if "abandoned" in p.stderr: print("abandoned:",it,kw,th,mb)
print("done",N,"bad",bad)
if record: print(json.dumps(digests))
sys.exit(1 if bad else 0)
