# per-phase cycle profile of the mix kernel (clock64 counters) on synthetic replay streams
import os, sys, time, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import cmix_b200
from conftest import synthetic_streams
n = int(sys.argv[1]) if len(sys.argv) > 1 else 512
stream, vocab, codes, ppmd = synthetic_streams(n, seed=1)
P = cmix_b200.Predictor(vocab)
P.code_bytes(stream[:64], codes[:512], ppmd[:64])       # warm-up
P.debug_fetch(6, (64,), np.uint64)                        # enable counters
t0 = time.time()
P.code_bytes(stream[64:], codes[512:], ppmd[64:])
dt = time.time() - t0
prof = P.debug_fetch(6, (64,), np.uint64).astype(np.float64)
bits = (n - 64) * 8
names = ['L pre', 'L bptt-recursion', 'L grad+adam', 'L out-SGD', 'L fwd stage', 'L fwd chain', 'L softmax', 'L fwd cluster.sync', 'L fwd cell+bcast', 'L fwd sums', 'L fwd norm+act']
print('wall %.3f s for %d bits = %.2f us/bit' % (dt, bits, dt / bits * 1e6))
prof8 = prof[8]
for i, nm in enumerate(names):
    print('%-18s %8.0f cycles/byte' % (nm, prof[32 + i] / bits * 8))
print('LSTM total         %8.0f cycles/byte' % (prof[32:43].sum() / bits * 8))
phases = {8:'C0 wait-ready',9:'C0 chain',10:'C0 recv',11:'C0 extras',12:'C0 coeff',13:'C0 publish',14:'C1 wait-ready',15:'C1 chain',16:'C1 recv',17:'C1 extras',18:'C1 coeff',19:'C1 publish',20:'M stage',21:'M aux+plan',22:'M jobs+rate',23:'M late path',24:'M wait-coeff',25:'M update',26:'T prefetch',27:'T wait-ring',28:'T layer1',29:'T layer2+SSE',30:'T update'}
for k in sorted(phases): print('%-18s %8.0f cycles/bit' % (phases[k], prof[k] / bits))
