# first GPU parity check against a dump generated on the box
import os, sys, subprocess, time, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tools'))
from oracle_io import Dump, N_EXT
import cmix_b200
from gen_synth import synth_text
os.makedirs('/tmp/w', exist_ok=True)
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1500
open('/tmp/w/s.txt','wb').write(synth_text(n))
t0=time.time()
subprocess.run([os.path.join(ROOT, 'oracle', '_ref', 'oracle_dump'),'dump','n','/tmp/w/s.txt','/tmp/w/d','2'], check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
print('oracle dump took', time.time()-t0)
d = Dump('/tmp/w/d')
t0=time.time()
P = cmix_b200.Predictor(d.vocab)
print('create took', time.time()-t0)
t0=time.time()
p = P.code_bytes(d.stream, d.ext, d.ppmd)
print('code_bytes took', time.time()-t0, 'for', d.n_bytes, 'bytes')
nb = d.n_bytes*8
sx = P.debug_fetch(1, (nb,56), np.float32)
sel = P.debug_fetch(2, (nb,48), np.uint32)
lx = P.debug_fetch(3, (nb,2), np.float32)
ref_small = np.concatenate([d.inputs[:, :3], d.inputs[:, 2025:2077]], axis=1)
bad = np.nonzero((sx[:, :55] != ref_small).any(axis=1))[0]
print('small_x mismatching bits:', len(bad), bad[:5])
if len(bad):
    t=bad[0]; w=np.nonzero(sx[t,:55]!=ref_small[t])[0]; print('  first bit', t, 'lanes', w, sx[t,w], ref_small[t,w])
cols=[i for i in range(47) if i!=12]
badc = np.nonzero((sel[:, cols] != d.ctx[:, cols]).any(axis=1))[0]
print('selector mismatching bits:', len(badc), badc[:5])
if len(badc):
    t=badc[0]; w=[c for c in cols if sel[t,c]!=d.ctx[t,c]]; print('  first bit', t, 'mixers', w, sel[t,w], d.ctx[t,w])
badl = np.nonzero(lx[:,0] != d.inputs[:,2077])[0]
print('lstm_x mismatching bits:', len(badl), badl[:5])
badp = np.nonzero(p != d.p)[0]
print('p mismatching bits:', len(badp), badp[:5], 'max abs diff', np.abs(p-d.p).max())
if len(badp): t=badp[0]; print('  first', t, p[t], d.p[t])
print('errflags', P.debug_fetch(5,(1,),np.uint32))
