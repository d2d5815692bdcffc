import os, sys, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import cmix_b200
from conftest import synthetic_streams
stream, vocab, codes, ppmd = synthetic_streams(40, seed=5)
P = cmix_b200.Predictor(vocab)
import time
t0=time.perf_counter()
for t in range(40*8):
    P.feed_external_bit(codes[t])
    p = P.Predict()
    if t % 8 == 7: P.feed_external_byte(ppmd[t//8])
    P.Perceive(int((stream[t>>3] >> (7-(t&7))) & 1))
print("us/bit", (time.perf_counter()-t0)/320*1e6)
P.close()
