"""Tuning-settings check: records extracted under different tuning settings must be identical (same set, bit for bit).
usage: variant_check.py key=a key=b ...   (first is the baseline)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import cudasift_b200 as cs
from cudasift_b200.synth import synth_image
cs.InitCuda(0)
FIELDS = ("xpos", "ypos", "scale", "sharpness", "edgeness", "orientation", "subsampling", "data")
def canon(p):
    return p[np.lexsort((p["orientation"], p["scale"], p["xpos"], p["ypos"], p["subsampling"]))]
def run(spec, img, octaves, thresh):
    for kv in spec.split(","):
        k, v = kv.split("="); cs.set_tuning(k, int(v))
    h, w = img.shape
    pitch = cs.iAlignUp(w, 128)
    ci = cs.CudaImage().Allocate(w, h, pitch, False, None, img); ci.Download()
    ex = cs.Extractor(w, h, octaves, 32768, False)
    ex.submit_device(ci.d_data, pitch, 1.0, thresh, 0.0)
    n = ex.wait()
    pts = ex.device_points_at(0, n)
    ex.close()
    return canon(pts)
specs = sys.argv[1:]
ok = True
for (w, h, o, t) in ((1920, 1080, 5, 3.0), (641, 479, 4, 2.0), (257, 131, 2, 1.5), (1000, 700, 7, 1.0)):
    img = synth_image(w, h, seed=1000 + w)
    base = run(specs[0], img, o, t)
    for sp in specs[1:]:
        got = run(sp, img, o, t)
        same = len(got) == len(base) and all(np.array_equal(got[f], base[f]) for f in FIELDS)
        print("%dx%d %s vs %s: %d / %d points %s" % (w, h, sp, specs[0], len(got), len(base), "IDENTICAL" if same else "DIFFERENT"), flush=True)
        ok = ok and same
sys.exit(0 if ok else 1)
