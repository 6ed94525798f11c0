import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import cudasift_b200 as cs
from cudasift_b200.synth import synth_image
cs.InitCuda(0)
w, h = 1920, 1080
pitch = cs.iAlignUp(w, 128)
imgs = [synth_image(w, h, seed=1000 + i) for i in range(8)]
cis = []
for i in range(32):
    ci = cs.CudaImage().Allocate(w, h, pitch, False, None, imgs[i % 8]); ci.Download(); cis.append(ci)
ptrs = [c.d_data for c in cis]
keys = sys.argv[1:] or ["d2_hs=0"]
for spec in keys:
    for kv in spec.split(","):
        k, v = kv.split("="); cs.set_tuning(k, int(v))
    for B in [int(x) for x in os.environ.get("R2_BATCHES", "1,32").split(",")]:
        ex = cs.Extractor(w, h, 5, 32768, False, batch=B)
        t = []
        for i in range(8):
            n, ms = ex.profile_batch(ptrs[:B], pitch, 1.0, 3.0, 0.0); t.append(ms)
        t = np.array(t[2:]).mean(axis=0) * 1e3 / B
        print("%-28s batch %2d per image: pyrA %.1f chain %.1f detect %.1f describe %.1f total %.1f us (%d pts/img)" % (spec, B, t[0], t[1], t[2], t[3], t[4], n // B), flush=True)
        ex.close()
