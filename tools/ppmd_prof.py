# per-phase cycle profile of the resident PPMD model (ppmd.cuh) on synthetic enwik-shaped text
import os, sys, time, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tools'))
import cmix_b200
from gen_synth import synth_text
n = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
data = np.frombuffer(synth_text(n, 0xE9E80021), dtype=np.uint8)
vocab = np.zeros(256, dtype=np.uint8); vocab[np.unique(data)] = 1
P = cmix_b200.Predictor(vocab)
t0 = time.time()
P.code_bytes(data, None, None)
dt = time.time() - t0
prof = P.debug_fetch(9, (6,), np.uint64).astype(np.float64)
names = ['symbol search', 'model update', 'suffix walk', 'ConvertSQ', 'emit']
print('wall %.3f s for %d bytes = %.1f us/byte (whole pipeline)' % (dt, n, dt / n * 1e6))
for i, nm in enumerate(names):
    print('%-14s %8.0f cycles/byte' % (nm, prof[i] / prof[5]))
print('PPMD total     %8.0f cycles/byte' % (prof[:5].sum() / prof[5]))
P.close()
